// generate.cu -- exl_gen_advance: the tail of one batched generation step in one launch (include/exl_b200.h).
//
// After the sampler has drawn one token per row, each row's request needs its history extended, its output rows written, its stop
// test made, the next step's input row gathered from the embedding table and the uniform of its next draw.  As torch ops that is a
// string of small launches per step; here it is one CTA per row, no atomics, and nothing the host has to wait for.  The status is
// sticky: once a slot has stopped or failed, later rows for it write nothing, so the host may step a finished row once more before
// it reads the status (exllama_b200/generate.py reads each step's status one step late).
#include "exl_common.cuh"
#include <cmath>

namespace {

constexpr int GA_THREADS = 128;

struct GenArgs {
    const int64_t* tokens; const float* probs;
    int slot[EXL_RAGGED_MAX_SEQ], pos[EXL_RAGGED_MAX_SEQ], j[EXL_RAGGED_MAX_SEQ];
    int64_t* hist; int64_t hist_ld; int* status; const int64_t* stop_ids; const uint64_t* seeds;
    const half* embed; int vocab, hidden; half* x_next; float* u_next;
    int64_t* out_tokens; float* out_probs; int64_t out_ld;
};
static_assert(sizeof(GenArgs) <= 4096, "GenArgs must fit the classic 4 KB kernel parameter space");

// U(seed, j) of include/exl_b200.h: output j of splitmix64 seeded with seed, top 24 bits over 2^24
__device__ float gen_uniform(uint64_t seed, int j)
{
    uint64_t x = seed + (uint64_t)(j + 1) * 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    x ^= x >> 31;
    return (float)(x >> 40) * (1.0f / 16777216.0f);
}

__global__ void __launch_bounds__(GA_THREADS) gen_advance_kernel(const __grid_constant__ GenArgs a)
{
    const int r = blockIdx.x;
    const int s = a.slot[r];
    if (s < 0) return;
    const int live = a.status[s] == EXL_GEN_LIVE;
    __syncthreads();                                                 // every thread has read the status before thread 0 may write it
    if (!live) return;
    const int64_t t = a.tokens[r];
    const int64_t o = (int64_t)s * a.out_ld + a.j[r];
    if (t < 0 || t >= a.vocab) {                                     // the sampler's undefined row
        if (threadIdx.x == 0) { a.out_tokens[o] = -1; a.out_probs[o] = NAN; a.status[s] = EXL_GEN_ERROR; }
        return;
    }
    if (threadIdx.x == 0) {
        a.hist[(int64_t)s * a.hist_ld + a.pos[r]] = t;
        a.out_tokens[o] = t;
        a.out_probs[o] = a.probs[r];
        bool stop = false;
        for (int k = 0; k < EXL_GEN_MAX_STOP; k++) stop |= a.stop_ids[(int64_t)s * EXL_GEN_MAX_STOP + k] == t;
        if (stop) a.status[s] = EXL_GEN_STOPPED;
        a.u_next[s] = gen_uniform(a.seeds[s], a.j[r] + 1);
    }
    const uint4* src = reinterpret_cast<const uint4*>(a.embed + t * a.hidden);
    uint4* dst = reinterpret_cast<uint4*>(a.x_next + (int64_t)s * a.hidden);
    for (int i = threadIdx.x; i < a.hidden / 8; i += GA_THREADS) dst[i] = src[i];
}

} // namespace

int exl_gen_advance_launch(const int64_t* tokens, const float* probs, int rows, const int* slot_host, const int* pos_host,
                           const int* j_host, int64_t* hist, int64_t hist_ld, int* status, const int64_t* stop_ids,
                           const uint64_t* seeds, int n_slots, const half* embed, int vocab, int hidden, half* x_next, float* u_next,
                           int64_t* out_tokens, float* out_probs, int64_t out_ld, cudaStream_t stream)
{
    if (rows < 1 || rows > EXL_RAGGED_MAX_SEQ) return exl_set_err(EXL_ERR_ARG, "gen_advance: rows %d outside [1, %d]", rows, EXL_RAGGED_MAX_SEQ);
    if (n_slots < 1 || n_slots > EXL_RAGGED_MAX_SEQ)
        return exl_set_err(EXL_ERR_ARG, "gen_advance: n_slots %d outside [1, %d]", n_slots, EXL_RAGGED_MAX_SEQ);
    if (vocab < 1) return exl_set_err(EXL_ERR_ARG, "gen_advance: vocab %d < 1", vocab);
    if (hidden < 8 || hidden % 8) return exl_set_err(EXL_ERR_ARG, "gen_advance: hidden %d is not a positive multiple of 8", hidden);
    if (!tokens || !probs || !slot_host || !pos_host || !j_host || !hist || !status || !stop_ids || !seeds || !embed || !x_next || !u_next ||
        !out_tokens || !out_probs)
        return exl_set_err(EXL_ERR_ARG, "gen_advance: NULL pointer");
    if (((uintptr_t)embed | (uintptr_t)x_next) & 15)
        return exl_set_err(EXL_ERR_ARG, "gen_advance: embed %p or x_next %p is not 16-byte aligned", (const void*)embed, (void*)x_next);
    GenArgs a{};
    bool seen[EXL_RAGGED_MAX_SEQ] = {};
    for (int r = 0; r < rows; r++) {
        const int s = slot_host[r];
        if (s < -1 || s >= n_slots) return exl_set_err(EXL_ERR_ARG, "gen_advance: row %d: slot %d outside [-1, n_slots %d)", r, s, n_slots);
        if (s >= 0) {
            if (seen[s]) return exl_set_err(EXL_ERR_ARG, "gen_advance: row %d: slot %d named twice", r, s);
            seen[s] = true;
            if (pos_host[r] < 0 || pos_host[r] >= hist_ld)
                return exl_set_err(EXL_ERR_ARG, "gen_advance: row %d: pos %d outside [0, hist_ld %lld)", r, pos_host[r], (long long)hist_ld);
            if (j_host[r] < 0 || j_host[r] >= out_ld)
                return exl_set_err(EXL_ERR_ARG, "gen_advance: row %d: j %d outside [0, out_ld %lld)", r, j_host[r], (long long)out_ld);
        }
        a.slot[r] = s; a.pos[r] = pos_host[r]; a.j[r] = j_host[r];
    }
    a.tokens = tokens; a.probs = probs;
    a.hist = hist; a.hist_ld = hist_ld; a.status = status; a.stop_ids = stop_ids; a.seeds = seeds;
    a.embed = embed; a.vocab = vocab; a.hidden = hidden; a.x_next = x_next; a.u_next = u_next;
    a.out_tokens = out_tokens; a.out_probs = out_probs; a.out_ld = out_ld;
    gen_advance_kernel<<<rows, GA_THREADS, 0, stream>>>(a);
    EXL_CHECK_LAUNCH("gen_advance_kernel");
    return EXL_OK;
}
