// gw-b200: kernels of the SSP chainer (chain_capi.cu, DESIGN.md section 19).
//
// The anchors are taken in ascending (q + t + L, index), the "rank" order: every predecessor of an anchor comes earlier in it.
// Ranks are cut into tiles of kTile. For each tile, chain_external_kernel tests every tile anchor against the anchors of all
// earlier tiles, one CTA per chunk of kChunk earlier anchors, and writes one (value, index) partial per (chunk, anchor);
// chain_tile_kernel then reduces those partials and walks the tile in rank order on one CTA: at step s, anchor s takes
// f = s + max(0, best) and every later tile anchor folds f(s) - pen(s, .) into its own best. A best is the largest value,
// ties to the smallest SSP index, so no partial depends on how the work is grouped.
#pragma once

#include <cstdint>

namespace gwb200
{
namespace chain
{

constexpr int kTile  = 1024; // anchors per tile = threads of chain_tile_kernel
constexpr int kChunk = 512;  // earlier anchors per CTA of chain_external_kernel
constexpr int kExternalThreads = 256;
constexpr int64_t kNone = INT64_MIN;

struct SspD
{
    uint32_t query, target;
    int32_t length, score;
};

// The rank-order view of the anchors: the ends + 1 of each (eq = q + L + 1, et = t + L + 1), its starts, score, SSP index and f.
struct Ranked
{
    int64_t* eq;
    int64_t* et;
    uint32_t* q;
    uint32_t* t;
    int32_t* s;
    int32_t* k;
    int64_t* f;
};

__device__ __forceinline__ bool better(int64_t v, int32_t i, int64_t bv, int32_t bi) { return v > bv || (v == bv && i < bi); }

// (value, index) of i -> j, or kNone when i does not precede j. dq, dt >= 0 is the precedence test.
__device__ __forceinline__ int64_t link(int64_t eq_i, int64_t et_i, int64_t f_i, int64_t q_j, int64_t t_j, int64_t D, int64_t A)
{
    const int64_t dq = q_j - eq_i, dt = t_j - et_i;
    if ((dq | dt) < 0)
        return kNone;
    const int64_t d = dt - dq;
    return f_i - D * (d < 0 ? -d : d) - A * (dq + dt);
}

// keys[k] = q + t + L + 1 (< 2^35), idx[k] = k; *bad = 1 when some length is below -1
__global__ void chain_keys_kernel(const SspD* __restrict__ ssps, int32_t n, uint64_t* __restrict__ keys, int32_t* __restrict__ idx,
                                  int32_t* __restrict__ bad)
{
    for (int32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    {
        const SspD a = ssps[k];
        if (a.length < -1)
            *bad = 1;
        keys[k] = uint64_t(int64_t(a.query) + a.target + a.length + 1);
        idx[k]  = k;
    }
}

__global__ void chain_stage_kernel(const SspD* __restrict__ ssps, const int32_t* __restrict__ order, int32_t n, Ranked r)
{
    for (int32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x)
    {
        const int32_t k = order[j];
        const SspD a    = ssps[k];
        r.eq[j]         = int64_t(a.query) + a.length + 1;
        r.et[j]         = int64_t(a.target) + a.length + 1;
        r.q[j]          = a.query;
        r.t[j]          = a.target;
        r.s[j]          = a.score;
        r.k[j]          = k;
    }
}

// grid (chunks of [0, first), ceil(m / kExternalThreads)): the best link from each chunk into tile anchors [first, first + m).
__global__ void __launch_bounds__(kExternalThreads) chain_external_kernel(Ranked r, int32_t first, int32_t m, int64_t D, int64_t A,
                                                                          int64_t* __restrict__ part_v, int32_t* __restrict__ part_i)
{
    __shared__ int64_t s_eq[kChunk], s_et[kChunk], s_f[kChunk];
    __shared__ int32_t s_k[kChunk];
    const int32_t c0 = blockIdx.x * kChunk;
    const int32_t cn = min(kChunk, first - c0);
    for (int32_t x = threadIdx.x; x < cn; x += blockDim.x)
    {
        s_eq[x] = r.eq[c0 + x];
        s_et[x] = r.et[c0 + x];
        s_f[x]  = r.f[c0 + x];
        s_k[x]  = r.k[c0 + x];
    }
    __syncthreads();
    const int32_t t = blockIdx.y * blockDim.x + threadIdx.x;
    if (t >= m)
        return;
    const int64_t qj = r.q[first + t], tj = r.t[first + t];
    int64_t bv = kNone;
    int32_t bi = INT32_MAX;
    for (int32_t x = 0; x < cn; ++x)
    {
        const int64_t v = link(s_eq[x], s_et[x], s_f[x], qj, tj, D, A);
        if (v != kNone && better(v, s_k[x], bv, bi))
            bv = v, bi = s_k[x];
    }
    part_v[int64_t(blockIdx.x) * kTile + t] = bv;
    part_i[int64_t(blockIdx.x) * kTile + t] = bi;
}

// One CTA of kTile threads: tile anchors [first, first + m) with `chunks` partials each; writes f in rank order and f, p by
// SSP index.
__global__ void __launch_bounds__(kTile) chain_tile_kernel(Ranked r, int32_t first, int32_t m, int32_t chunks, int64_t D, int64_t A,
                                                           const int64_t* __restrict__ part_v, const int32_t* __restrict__ part_i,
                                                           int64_t* __restrict__ f_out, int32_t* __restrict__ p_out)
{
    __shared__ int64_t b_eq[2], b_et[2], b_f[2];
    __shared__ int32_t b_k[2];
    const int32_t t = threadIdx.x;
    const bool live = t < m;
    int64_t bv = kNone, qj = 0, tj = 0;
    int32_t bi = INT32_MAX, kj = 0;
    if (live)
    {
        for (int32_t c = 0; c < chunks; ++c)
        {
            const int64_t v = part_v[int64_t(c) * kTile + t];
            const int32_t i = part_i[int64_t(c) * kTile + t];
            if (v != kNone && better(v, i, bv, bi))
                bv = v, bi = i;
        }
        qj = r.q[first + t];
        tj = r.t[first + t];
        kj = r.k[first + t];
    }
    for (int32_t s = 0; s < m; ++s)
    {
        const int b = s & 1;
        if (t == s)
        {
            const bool linked = bv > 0;
            const int64_t f   = r.s[first + t] + (linked ? bv : 0);
            r.f[first + t]    = f;
            f_out[kj]         = f;
            p_out[kj]         = linked ? bi : -1;
            b_eq[b]           = r.eq[first + t];
            b_et[b]           = r.et[first + t];
            b_f[b]            = f;
            b_k[b]            = kj;
        }
        __syncthreads();
        if (t > s && live)
        {
            const int64_t v = link(b_eq[b], b_et[b], b_f[b], qj, tj, D, A);
            if (v != kNone && better(v, b_k[b], bv, bi))
                bv = v, bi = b_k[b];
        }
    }
}

// One CTA: the end (largest f, ties to the smallest index), then the chain flagged by following p from it on one thread.
// res[0] = chain length, res[1] = its score.
__global__ void __launch_bounds__(1024) chain_finish_kernel(const int64_t* __restrict__ f, const int32_t* __restrict__ p, int32_t n,
                                                            uint8_t* __restrict__ flags, int64_t* __restrict__ res)
{
    __shared__ int64_t w_v[32];
    __shared__ int32_t w_i[32];
    int64_t bv = kNone;
    int32_t bi = INT32_MAX;
    for (int32_t k = threadIdx.x; k < n; k += blockDim.x)
        if (better(f[k], k, bv, bi))
            bv = f[k], bi = k;
    for (int o = 16; o > 0; o >>= 1)
    {
        const int64_t v = __shfl_down_sync(0xffffffffu, bv, o);
        const int32_t i = __shfl_down_sync(0xffffffffu, bi, o);
        if (better(v, i, bv, bi))
            bv = v, bi = i;
    }
    if ((threadIdx.x & 31) == 0)
        w_v[threadIdx.x >> 5] = bv, w_i[threadIdx.x >> 5] = bi;
    __syncthreads();
    if (threadIdx.x != 0)
        return;
    for (int w = 1; w < int(blockDim.x >> 5); ++w)
        if (better(w_v[w], w_i[w], bv, bi))
            bv = w_v[w], bi = w_i[w];
    int64_t len = 0;
    for (int32_t k = bi; k >= 0; k = p[k])
    {
        flags[k] = 1;
        ++len;
    }
    res[0] = len;
    res[1] = bv;
}

// ---- every chain above a minimum score (DESIGN.md section 20), on top of the f and p above ----

constexpr int kClaimThreads      = 1024;
constexpr int32_t kClaimStagedMax = 28 * 1024; // SSPs whose p and owner marks (8 bytes each, 224 KiB) fit in shared memory

// The priority order is f descending, ties to the smallest index: an ascending key ~(f with its sign bit flipped), sorted stably
// with idx[k] = k.
__global__ void chain_priority_keys_kernel(const int64_t* __restrict__ f, int32_t n, uint64_t* __restrict__ keys, int32_t* __restrict__ idx)
{
    for (int32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    {
        keys[k] = ~(uint64_t(f[k]) ^ (uint64_t(1) << 63));
        idx[k]  = k;
    }
}

// One CTA: the claim walk. order[r] is the SSP of priority rank r. Every unclaimed SSP h, in priority order, heads chain c (the
// next ordinal): h, p(h), p(p(h)), ... are claimed (owner = c) up to -1 or the first SSP already claimed. With `staged`, p and the
// owner marks live in 8n bytes of dynamic shared memory; otherwise in global memory. Warp 0 reads the next 32 ranks and their
// marks at once; a mark seen as claimed stays claimed, so only the open ones are re-read by the walking lane.
__global__ void __launch_bounds__(kClaimThreads) chain_claim_kernel(const int32_t* __restrict__ order, const int32_t* p_g, int32_t n, int32_t staged,
                                                                    int32_t* owner_g, int32_t* __restrict__ heads, int32_t* __restrict__ count)
{
    extern __shared__ int32_t smem[];
    __shared__ int32_t batch[32];
    const int32_t* p = p_g;
    int32_t* owner   = owner_g;
    if (staged)
    {
        p     = smem;
        owner = smem + n;
        for (int32_t x = threadIdx.x; x < n; x += blockDim.x)
            smem[x] = p_g[x];
    }
    for (int32_t x = threadIdx.x; x < n; x += blockDim.x)
        owner[x] = -1;
    __syncthreads();
    if (threadIdx.x < 32)
    {
        const int lane = threadIdx.x;
        int32_t c      = 0;
        for (int32_t r0 = 0; r0 < n; r0 += 32)
        {
            const int32_t h    = r0 + lane < n ? order[r0 + lane] : -1;
            unsigned open      = __ballot_sync(0xffffffffu, h >= 0 && owner[h] < 0);
            batch[lane]        = h;
            __syncwarp();
            if (lane == 0)
                while (open)
                {
                    int32_t k = batch[__ffs(open) - 1];
                    open &= open - 1;
                    if (owner[k] >= 0)
                        continue;
                    heads[c] = k;
                    for (; k >= 0 && owner[k] < 0; k = p[k])
                        owner[k] = c;
                    ++c;
                }
            __syncwarp();
        }
        if (lane == 0)
            *count = c;
    }
    __syncthreads();
    if (staged)
        for (int32_t x = threadIdx.x; x < n; x += blockDim.x)
            owner_g[x] = owner[x];
}

// One thread per SSP. k is the first member of its chain c when p(k) = -1 or p(k) belongs to another chain; exactly one member
// is, and it writes the chain's score f(head) - f(k) + s(k). len[c] counts the members (zeroed before).
__global__ void chain_score_kernel(const SspD* __restrict__ ssps, const int64_t* __restrict__ f, const int32_t* __restrict__ p,
                                   const int32_t* __restrict__ owner, const int32_t* __restrict__ heads, int32_t n, int64_t* __restrict__ score,
                                   int32_t* __restrict__ len)
{
    for (int32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    {
        const int32_t c = owner[k], pk = p[k];
        atomicAdd(&len[c], 1);
        if (pk < 0 || owner[pk] != c)
            score[c] = f[heads[c]] - f[k] + ssps[k].score;
    }
}

// One thread per SSP and per chain. member[k]: k's chain is kept (score >= S); skey[k] = its chain for a member, n otherwise, and
// sval[k] = k, for the stable sort into (chain, index). keep[c] for c < *count (zero beyond), and the kept scores summed into *sum.
__global__ void chain_keep_kernel(const int32_t* __restrict__ owner, const int64_t* __restrict__ score, const int32_t* __restrict__ count, int32_t n,
                                  int64_t S, uint8_t* __restrict__ member, uint8_t* __restrict__ keep, uint32_t* __restrict__ skey,
                                  int32_t* __restrict__ sval, unsigned long long* __restrict__ sum)
{
    const int32_t chains = *count;
    for (int32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    {
        const int32_t c = owner[k];
        const bool m    = score[c] >= S;
        member[k]       = m;
        skey[k]         = uint32_t(m ? c : n);
        sval[k]         = k;
        const bool kc   = k < chains && score[k] >= S;
        keep[k]         = kc;
        if (kc)
            atomicAdd(sum, static_cast<unsigned long long>(score[k])); // mod 2^64: the int64 sum in any order
    }
}

} // namespace chain
} // namespace gwb200
