"""The one loader of the checkers the tests compare the engine against: the CPU restatements oracle/lib*.so (built by
oracle/Makefile) and the libraries of the unmodified reference under oracle/_ref/, and the gzip JSON fixtures under
tests/golden/. Also the one device allocator the GPU tests hand to the engines to check that their memory balances. TEST
INFRASTRUCTURE ONLY."""
import ctypes as C
import gzip
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
REF_DIR = os.path.join(ORACLE_DIR, "_ref")
GOLDEN = os.path.join(ROOT, "tests", "golden")
if ROOT not in sys.path:  # the checkers' modules use genomeworks_b200, also when a fixture maker runs them
    sys.path.insert(0, ROOT)

_loaded = {}


def ptr(a):
    """The address of a numpy array as a c_void_p; None for None."""
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def load(name, signatures):
    """The library oracle/<name>, loaded once per process, with each function of `signatures`, {function: (restype, argtypes)},
    declared. A CPU checker ("lib*.so") is first brought up to date by `make -C oracle <name>`, so that a test never runs
    against a build older than the checker's sources; a reference library ("_ref/...") is only loaded."""
    if name not in _loaded:
        if os.path.dirname(name) == "":
            subprocess.check_call(["make", "-C", ORACLE_DIR, name], stdout=subprocess.DEVNULL)
        lib = C.CDLL(os.path.join(ORACLE_DIR, name))
        for f, (restype, argtypes) in signatures.items():
            getattr(lib, f).restype = restype
            getattr(lib, f).argtypes = argtypes
        _loaded[name] = lib
    return _loaded[name]


def read_fixture(path):
    with gzip.open(path, "rt") as f:
        return json.load(f)


def write_fixture(path, obj):
    """obj as gzip JSON with sorted keys; the gzip header carries no timestamp, so equal content gives equal bytes."""
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with gzip.GzipFile(path, "wb", mtime=0) as f:
        f.write(json.dumps(obj, sort_keys=True).encode())


class CountingAllocator:
    """Device memory from torch's caching allocator; counts the requests, keeps the size of each block outstanding, checks
    that a block is freed with its size, and can refuse its n-th request."""

    def __init__(self, refuse=None):
        import torch
        self.torch = torch
        self.live = {}
        self.calls = 0
        self.refuse = refuse

    def alloc(self, n):
        self.calls += 1
        if self.calls == self.refuse:
            return 0
        p = self.torch.cuda.caching_allocator_alloc(int(n))
        self.live[p] = n
        return p

    def free(self, p, n):
        assert self.live.pop(p) == n
        self.torch.cuda.caching_allocator_delete(p)
