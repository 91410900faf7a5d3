"""Checkers of the SSP chainer (DESIGN.md section 19): ctypes bindings for its CPU oracle (oracle/liboracle_chain.so), a plain-
Python restatement of the contract that pins the oracle, SSP set generators and a check of the contract's equations on the
device. TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import functools
import sys

import numpy as np

from checker_lib import load, ptr
from extender_libs import SSP_DTYPE

MAX_PENALTY = 1 << 20


def oracle():
    return load("liboracle_chain.so", {
        "oracle_chain_run": (C.c_int64, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p])})


def oracle_run(ssps, D=0, A=0):
    """{f, p, chain (e, p(e), ...), score} of the contract over an SSP_DTYPE array."""
    s = np.ascontiguousarray(ssps, dtype=SSP_DTYPE)
    n = len(s)
    f = np.zeros(n, dtype=np.int64)
    p = np.zeros(n, dtype=np.int32)
    chain = np.zeros(max(n, 1), dtype=np.int32)
    score = C.c_int64()
    m = oracle().oracle_chain_run(ptr(s), n, D, A, ptr(f), ptr(p), ptr(chain), C.byref(score))
    if m < 0:
        raise ValueError("an SSP length is below -1")
    return {"f": f, "p": p, "chain": chain[:m].copy(), "score": score.value}


def chain_indices(res):
    """The chain's SSP indices in ascending order, as the engine returns them."""
    return np.sort(res["chain"]).astype(np.int32)


def python_chain(ssps, D=0, A=0):
    """The contract restated: precedence tested pair by pair, f by memoised recursion over the predecessors (no evaluation order
    is assumed), the end and the chain as defined."""
    rows = [(int(r["query"]), int(r["target"]), int(r["length"]), int(r["score"])) for r in ssps]
    n = len(rows)

    def before(i, j):
        qi, ti, li, _ = rows[i]
        qj, tj, _, _ = rows[j]
        return ti + li < tj and qi + li < qj

    def precedes(i, j):
        return before(i, j) and (not before(j, i) or i < j)

    preds = [[i for i in range(n) if i != j and precedes(i, j)] for j in range(n)]
    sys.setrecursionlimit(max(sys.getrecursionlimit(), 4 * n + 100))

    @functools.lru_cache(maxsize=None)
    def fp(j):
        qj, tj, _, sj = rows[j]
        best, arg = 0, -1
        for i in preds[j]:
            qi, ti, li, _ = rows[i]
            dq, dt = qj - qi - li - 1, tj - ti - li - 1
            v = fp(i)[0] - (D * abs(dt - dq) + A * (dq + dt))
            if v > best:  # ascending i: the first to attain the maximum is kept
                best, arg = v, i
        return sj + best, arg

    f = np.array([fp(j)[0] for j in range(n)], dtype=np.int64)
    p = np.array([fp(j)[1] for j in range(n)], dtype=np.int32)
    if n == 0:
        return {"f": f, "p": p, "chain": np.zeros(0, dtype=np.int32), "score": 0}
    e = int(np.flatnonzero(f == f.max())[0])
    chain = [e]
    while p[chain[-1]] >= 0:
        chain.append(int(p[chain[-1]]))
    return {"f": f, "p": p, "chain": np.array(chain, dtype=np.int32), "score": int(f[e])}


def same(a, b):
    return np.array_equal(a["f"], b["f"]) and np.array_equal(a["p"], b["p"]) and np.array_equal(a["chain"], b["chain"]) and \
        a["score"] == b["score"]


def ssps_of(rows):
    out = np.zeros(len(rows), dtype=SSP_DTYPE)
    for k, r in enumerate(rows):
        out[k] = r
    return out


def random_ssps(rng, n, span=300, max_len=30, scores=(-20, 60), base=0):
    """n random SSPs with starts in [base, base + span), lengths in [-1, max_len] and scores in `scores`: dense enough for many
    links, equal values and touching or overlapping segments."""
    s = np.zeros(n, dtype=SSP_DTYPE)
    s["query"] = base + rng.integers(0, span, n)
    s["target"] = base + rng.integers(0, span, n)
    s["length"] = rng.integers(-1, max_len + 1, n)
    s["score"] = rng.integers(scores[0], scores[1] + 1, n)
    return s


def ladder(n, step=50, length=30, score=100):
    """n colinear SSPs on one diagonal, each ending before the next begins: with zero penalties the chain is all of them."""
    s = np.zeros(n, dtype=SSP_DTYPE)
    s["query"] = np.arange(n) * step
    s["target"] = np.arange(n) * step + 7
    s["length"] = length
    s["score"] = score
    return s


def anti_diagonal(n, length=30, score=100):
    """n SSPs along one anti-diagonal (query rising as target falls): no two chain, so the chain is one SSP."""
    s = np.zeros(n, dtype=SSP_DTYPE)
    s["query"] = np.arange(n) * 40
    s["target"] = (n - 1 - np.arange(n)) * 40
    s["length"] = length
    s["score"] = score
    return s


def backbone_set(rng, n, backbone, span=10 ** 8):
    """n SSPs: a colinear backbone of `backbone` SSPs with jittered gaps and diagonals, and n - backbone random off-chain SSPs
    over the same span, in a shuffled order."""
    s = np.zeros(n, dtype=SSP_DTYPE)
    step = span // max(backbone, 1)
    q0 = np.arange(backbone, dtype=np.int64) * step
    s["query"][:backbone] = q0 + rng.integers(0, step // 4, backbone)
    s["target"][:backbone] = q0 + rng.integers(0, step // 4, backbone)
    s["length"][:backbone] = rng.integers(20, min(200, step // 2), backbone)
    s["score"][:backbone] = rng.integers(3000, 20000, backbone)
    m = n - backbone
    s["query"][backbone:] = rng.integers(0, span, m)
    s["target"][backbone:] = rng.integers(0, span, m)
    s["length"][backbone:] = rng.integers(20, 200, m)
    s["score"][backbone:] = rng.integers(3000, 20000, m)
    return s[rng.permutation(n)]


def check_contract_on_device(ssps, D, A, f, p, chain, score, rows_per_step=256, device="cuda"):
    """The contract's equations for a device result at sizes the O(n^2) oracle is too slow for, evaluated with torch on the GPU:
    f(j) = s_j + max(0, best_j) and p(j) the smallest index attaining best_j > 0, for every j, then the end and the chain. f is
    the unique solution of these equations, so this is the oracle's answer. One step holds a few int64 tensors of
    rows_per_step x n elements (200 MB each at n = 10^5)."""
    import torch
    dev = torch.device(device)
    q = torch.from_numpy(ssps["query"].astype(np.int64)).to(dev)
    t = torch.from_numpy(ssps["target"].astype(np.int64)).to(dev)
    L = torch.from_numpy(ssps["length"].astype(np.int64)).to(dev)
    s = torch.from_numpy(ssps["score"].astype(np.int64)).to(dev)
    fd = torch.from_numpy(np.asarray(f, np.int64)).to(dev)
    n = len(ssps)
    idx = torch.arange(n, device=dev)
    none = torch.iinfo(torch.int64).min
    for j0 in range(0, n, rows_per_step):
        j = idx[j0:j0 + rows_per_step, None]
        dq, dt = q[j] - q[None] - L[None] - 1, t[j] - t[None] - L[None] - 1
        before_ij = (dq >= 0) & (dt >= 0)
        before_ji = (q[None] - q[j] - L[j] - 1 >= 0) & (t[None] - t[j] - L[j] - 1 >= 0)
        pre = before_ij & (~before_ji | (idx[None] < j))
        v = torch.where(pre, fd[None] - D * (dt - dq).abs() - A * (dq + dt), torch.full_like(dq, none))
        best = v.max(dim=1).values
        linked = best > 0
        want_f = s[j0:j0 + rows_per_step] + torch.where(linked, best, torch.zeros_like(best))
        first = torch.where(v == best[:, None], idx[None].expand_as(v), torch.full_like(v, n)).min(dim=1).values
        want_p = torch.where(linked, first, torch.full_like(first, -1))
        assert torch.equal(want_f, fd[j0:j0 + rows_per_step]), j0
        assert torch.equal(want_p.cpu(), torch.from_numpy(np.asarray(p[j0:j0 + rows_per_step], np.int64))), j0
    e = int(np.flatnonzero(f == f.max())[0])
    walk = [e]
    while p[walk[-1]] >= 0:
        walk.append(int(p[walk[-1]]))
    assert score == int(f[e]) and np.array_equal(np.sort(walk), chain)
