// sample_select.cuh -- the sampler's order keys and radix selector (csrc/sample.cu), shared with csrc/beam.cu.
//
// One thread-block cluster of SP_CL CTAs per row; CTA r keeps the slice [r * slice, (r + 1) * slice) of the row in shared memory.
// Tokens are ordered by 50-bit keys (the float's bits above the inverted token id, so keys are unique and a tie goes to the lower
// id); radix_descent finds the key of a given rank, or the first key whose inclusive mass crosses a threshold, over the cluster in
// five 10-bit digits with bucket histograms -- no sort.  Every CTA reads the same merged values in the same order and so takes
// the same decisions.
#pragma once
#include "exl_common.cuh"
#include <cooperative_groups.h>

namespace {

namespace cg = cooperative_groups;

constexpr int SP_CL = 8;                        // CTAs per row
constexpr int SP_THREADS = 512;
constexpr int SP_MAX_VOCAB = 262144;            // token ids fit SP_ID_BITS
constexpr int SP_ID_BITS = 18;
constexpr int SP_DIGIT = 10;
constexpr int SP_BINS = 1 << SP_DIGIT;
constexpr int SP_KEY_BITS = 50;                 // 32-bit float field above the 18-bit id field
constexpr int SP_PASSES = SP_KEY_BITS / SP_DIGIT;
constexpr int SP_VTAB = 2048;                   // penalty recurrence values kept in shared memory (longer chains continue in registers)
constexpr int SP_MAX_SLICE = (SP_MAX_VOCAB + SP_CL - 1) / SP_CL;
constexpr double SP_FIX = 1152921504606846976.0;   // 2^60: probability mass in fixed point
static_assert(SP_PASSES * SP_DIGIT == SP_KEY_BITS, "whole digits");
static_assert(SP_MAX_VOCAB <= (1 << SP_ID_BITS), "ids fit the key's id field");
static_assert(2 * SP_BINS == 4 * SP_THREADS, "each thread scans two bins");

struct Part { float f; int bad; unsigned c; unsigned long long m; };

struct Shared {
    unsigned cnt[2][SP_BINS];
    unsigned long long mass[2][SP_BINS];
    float vtab[SP_VTAB];
    Part xch[2];                 // this CTA's contribution to the last two cluster exchanges
    Part bc;                     // merged result, broadcast to the block
    float redf[SP_THREADS / 32];
    unsigned long long redm[SP_THREADS / 32];
    unsigned redc[SP_THREADS / 32];
    int redi[SP_THREADS / 32];
    int found_pos;
    unsigned long long found_excl_m; unsigned found_excl_c;
};

__device__ __forceinline__ unsigned long long fix60(float w) { return __float2ull_rz(w * 0x1p60f); }

// order keys: larger key = earlier in the order; the low SP_ID_BITS hold the inverted id, so a tie goes to the lower id
__device__ __forceinline__ unsigned long long desc_key(float v, int id)
{
    return ((unsigned long long)__float_as_uint(v) << SP_ID_BITS) | (unsigned)((SP_MAX_VOCAB - 1) - id);
}
__device__ __forceinline__ unsigned long long asc_key(float v, int id)
{
    return ((unsigned long long)(0xFFFFFFFFu - __float_as_uint(v)) << SP_ID_BITS) | (unsigned)((SP_MAX_VOCAB - 1) - id);
}

// one fixed-order block reduction: warp butterflies, then warp 0 over the warp results
__device__ float block_sum_f(float v, Shared& sh)
{
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh.redf[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = 0.f;
    if (threadIdx.x == 0) for (int w = 0; w < SP_THREADS / 32; w++) s += sh.redf[w];
    return s;                                                        // valid in thread 0
}
__device__ float block_max_f(float v, Shared& sh)
{
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh.redf[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = -INFINITY;
    if (threadIdx.x == 0) for (int w = 0; w < SP_THREADS / 32; w++) s = fmaxf(s, sh.redf[w]);
    return s;
}
__device__ unsigned block_sum_c(unsigned v, Shared& sh)
{
    v = __reduce_add_sync(0xffffffffu, v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh.redc[threadIdx.x >> 5] = v;
    __syncthreads();
    unsigned s = 0;
    if (threadIdx.x == 0) for (int w = 0; w < SP_THREADS / 32; w++) s += sh.redc[w];
    return s;
}
__device__ int block_or(int v, Shared& sh)
{
    v = __any_sync(0xffffffffu, v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh.redi[threadIdx.x >> 5] = v;
    __syncthreads();
    int s = 0;
    if (threadIdx.x == 0) for (int w = 0; w < SP_THREADS / 32; w++) s |= sh.redi[w];
    return s;
}

// Cluster exchange: thread 0's `mine` goes to every CTA; thread 0 combines the SP_CL parts in rank order (combine(parts, out))
// and the result lands in sh.bc for the whole block.  One cluster barrier per exchange; the parity of `ph` alternates the
// exchange slots and histogram buffers, so a slot is rewritten only after every CTA has passed the barrier that follows its read.
template <class Combine>
__device__ void cluster_exchange(Shared& sh, int& ph, const Part& mine, Combine combine)
{
    cg::cluster_group cluster = cg::this_cluster();
    if (threadIdx.x == 0) sh.xch[ph & 1] = mine;
    cluster.sync();
    if (threadIdx.x == 0) {
        Part parts[SP_CL];
#pragma unroll
        for (int r = 0; r < SP_CL; r++) parts[r] = *cluster.map_shared_rank(&sh.xch[ph & 1], r);
        combine(parts, sh.bc);
    }
    __syncthreads();
    ph++;
}

__device__ float cluster_sum_f(Shared& sh, int& ph, float v)
{
    Part p{}; p.f = block_sum_f(v, sh);
    cluster_exchange(sh, ph, p, [](const Part* ps, Part& o) { float s = 0.f; for (int r = 0; r < SP_CL; r++) s += ps[r].f; o.f = s; });
    return sh.bc.f;
}
__device__ unsigned cluster_sum_c(Shared& sh, int& ph, unsigned v)
{
    Part p{}; p.c = block_sum_c(v, sh);
    cluster_exchange(sh, ph, p, [](const Part* ps, Part& o) { unsigned s = 0; for (int r = 0; r < SP_CL; r++) s += ps[r].c; o.c = s; });
    return sh.bc.c;
}

// The row's filter state: each stage's cut (a key threshold; 0 keeps everything) and normaliser (1 until the stage has run, and for
// a stage that is off: x / 1.0f is x, bit for bit).
struct Row {
    unsigned long long kk = 0, kp = 0, kt = 0;
    float sk = 1.0f, sp = 1.0f, st = 1.0f, negent = 0.0f;
};

// One token after the stages up to `level` (1: top-k, 2: top-p, 3: typical): whether it is kept, its key in that level's order
// and its probability there.
struct Tok { bool in; unsigned long long key; float w; };

__device__ __forceinline__ Tok eval(const Row& R, float p, int id, int level)
{
    Tok t;
    t.key = desc_key(p, id);
    t.in = t.key >= R.kk;
    const float q = p / R.sk;
    t.w = q;
    if (level < 2) return t;
    t.in = t.in && t.key >= R.kp;
    const float r = q / R.sp;
    t.w = r;
    if (level < 3) return t;
    const float d = fabsf(R.negent - logf(r + 1e-10f));
    t.key = asc_key(d, id);
    t.in = t.in && t.key >= R.kt;
    t.w = r / R.st;
    return t;
}

struct Descent { unsigned long long key; unsigned before; bool found; };

// Radix descent over the keys of the tokens `in` at `level`, in decreasing key order.
//   cross == false: the token of rank k (1-based).
//   cross == true : the first token whose inclusive mass (fixed point, weights w) exceeds T.
__device__ Descent radix_descent(Shared& sh, int& ph, const Row& R, const float* s_row, int n, int lo, int level, bool cross,
                                 unsigned k, unsigned long long T)
{
    cg::cluster_group cluster = cg::this_cluster();
    unsigned long long prefix = 0, acc = 0;
    unsigned before = 0;
    for (int pass = 0; pass < SP_PASSES; pass++) {
        const int shift = SP_KEY_BITS - SP_DIGIT * (pass + 1);
        const int buf = ph & 1;
        for (int b = threadIdx.x; b < SP_BINS; b += SP_THREADS) { sh.cnt[buf][b] = 0; sh.mass[buf][b] = 0; }
        if (threadIdx.x == 0) sh.found_pos = -1;
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += SP_THREADS) {
            const Tok t = eval(R, s_row[i], lo + i, level);
            if (!t.in || (t.key >> (shift + SP_DIGIT)) != (prefix >> (shift + SP_DIGIT))) continue;
            const int d = (int)(t.key >> shift) & (SP_BINS - 1);
            atomicAdd(&sh.cnt[buf][d], 1u);
            if (cross) atomicAdd(&sh.mass[buf][d], fix60(t.w));
        }
        cluster.sync();
        // positions 2t, 2t + 1 of the descending bin order (bins SP_BINS-1-2t, SP_BINS-2-2t), merged over the cluster
        unsigned c[2] = {0, 0}; unsigned long long m[2] = {0, 0};
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const int bin = SP_BINS - 1 - (2 * threadIdx.x + e);
#pragma unroll
            for (int r = 0; r < SP_CL; r++) {
                c[e] += cluster.map_shared_rank(&sh.cnt[buf][0], r)[bin];
                if (cross) m[e] += cluster.map_shared_rank(&sh.mass[buf][0], r)[bin];
            }
        }
        // block inclusive scan of the pairs
        unsigned cs = c[0] + c[1]; unsigned long long ms = m[0] + m[1];
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        unsigned ci = cs; unsigned long long mi = ms;
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned cu = __shfl_up_sync(0xffffffffu, ci, o);
            const unsigned long long mu = __shfl_up_sync(0xffffffffu, mi, o);
            if (lane >= o) { ci += cu; mi += mu; }
        }
        if (lane == 31) { sh.redc[warp] = ci; sh.redm[warp] = mi; }
        __syncthreads();
        unsigned cb = ci - cs; unsigned long long mb = mi - ms;
        for (int w = 0; w < warp; w++) { cb += sh.redc[w]; mb += sh.redm[w]; }
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const unsigned c_incl = cb + c[e]; const unsigned long long m_incl = mb + m[e];
            const bool hit = cross ? (acc + mb <= T && acc + m_incl > T) : (cb < k && k <= c_incl);
            if (hit) { sh.found_pos = 2 * threadIdx.x + e; sh.found_excl_c = cb; sh.found_excl_m = mb; }
            cb = c_incl; mb = m_incl;
        }
        __syncthreads();
        const int pos = sh.found_pos;
        ph++;
        if (pos < 0) return Descent{0, 0, false};                    // the same decision in every CTA
        prefix |= (unsigned long long)(SP_BINS - 1 - pos) << shift;
        before += sh.found_excl_c;
        acc += sh.found_excl_m;
        if (!cross) k -= sh.found_excl_c;
        __syncthreads();                                             // sh.found_* are rewritten by the next pass
    }
    return Descent{prefix, before, true};
}

} // namespace
