// toplp.cu -- exl_top_logprobs: the model's log-probability of each row's chosen token and its top-N alternatives, on the fp32
// logits the sampler reads (include/exl_b200.h).
//
// Layout     one thread-block cluster of SP_CL CTAs per row with the sampler's slices (csrc/sample_select.cuh): CTA r keeps the slice
//            [r * slice, (r + 1) * slice) of the row in shared memory.  The maximum, the undefined flag and the count of finite
//            entries are merged in one cluster exchange; the float64 exp-sum in a second (cluster_sum_d: threads, warps, CTAs in a
//            fixed order).
// Top-N      each finite logit gets a 50-bit key: the float's bits under the sign flip (-0 read as +0) above the inverted id, so keys
//            are unique, larger logits come first and a tie goes to the lower id.  The sampler's radix_descent finds the key of rank
//            K = min(N, #finite); each CTA lists its entries at or above it (exactly K in the cluster), and each listed entry's rank
//            is the number of listed keys above its own, read over distributed shared memory.  No sort, no floating-point atomics:
//            two calls are bitwise equal.
// Routing    with slot_host, row r writes output row [slot][j] only while status[slot] is EXL_GEN_LIVE (exl_gen_advance's gate),
//            so batched generation launches it between the sampler and the advance without waiting on the device.
#include "sample_select.cuh"
#include <cmath>

namespace {

struct TopArgs {
    const float* logits; int64_t ld; int vocab; int slice;
    const int64_t* tokens;                       // [rows] or NULL
    int n_top; int64_t top_ld;
    const int* status; int64_t out_ld;           // status NULL: row r writes output row r
    float* lp; int64_t* ids; float* top;
    int slot[EXL_RAGGED_MAX_SEQ], j[EXL_RAGGED_MAX_SEQ];
};
static_assert(sizeof(TopArgs) <= 4096, "TopArgs must fit the classic 4 KB kernel parameter space");

// the order key of a finite logit: the float's bits made monotone (sign flip; -0 canonicalised to +0) above the inverted id
__device__ __forceinline__ unsigned long long logit_key(float x, int id)
{
    const unsigned u = __float_as_uint(x == 0.0f ? 0.0f : x);
    const unsigned m = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ((unsigned long long)m << SP_ID_BITS) | (unsigned)((SP_MAX_VOCAB - 1) - id);
}

// radix_descent's evaluator over logits: every finite entry is in, keyed by logit_key
struct LogitEval {
    __device__ __forceinline__ Tok operator()(float x, int id) const
    {
        Tok t;
        t.in = isfinite(x);
        t.key = logit_key(x, id);
        t.w = 0.0f;
        return t;
    }
};

__global__ void __cluster_dims__(SP_CL, 1, 1) __launch_bounds__(SP_THREADS, 1) top_logprobs_kernel(const __grid_constant__ TopArgs a)
{
    extern __shared__ __align__(16) float s_row[];
    __shared__ Shared sh;
    __shared__ unsigned long long s_key[EXL_TOPLP_MAX];  // this CTA's entries at or above the rank-K key
    __shared__ float s_val[EXL_TOPLP_MAX];
    __shared__ unsigned s_cnt;
    cg::cluster_group cluster = cg::this_cluster();
    const int row = blockIdx.y;
    const int rank = (int)cluster.block_rank();
    const int lo = rank * a.slice;
    const int n = max(0, min(a.slice, a.vocab - lo));
    int64_t o = row;                                                 // output row
    if (a.status) {
        const int s = a.slot[row];
        if (s < 0 || a.status[s] != EXL_GEN_LIVE) return;            // the same value in every CTA of the cluster: no exchange yet
        o = (int64_t)s * a.out_ld + a.j[row];
    }
    int ph = 0;

    // 1. the slice into shared memory; the maximum finite entry, the undefined test (NaN or +inf), the count of finite entries
    const float* lg = a.logits + (int64_t)row * a.ld + lo;
    float mx = -INFINITY;
    int bad = 0;
    unsigned fin = 0;
    for (int i = threadIdx.x; i < n; i += SP_THREADS) {
        const float x = lg[i];
        s_row[i] = x;
        bad |= isnan(x) || x == INFINITY;
        if (isfinite(x)) { mx = fmaxf(mx, x); fin++; }
    }
    {
        Part p{}; p.f = block_max_f(mx, sh); p.bad = block_or(bad, sh); p.c = block_sum_c(fin, sh);
        cluster_exchange(sh, ph, p, [](const Part* ps, Part& q) {
            float m = -INFINITY; int b = 0; unsigned c = 0;
            for (int r = 0; r < SP_CL; r++) { m = fmaxf(m, ps[r].f); b |= ps[r].bad; c += ps[r].c; }
            q.f = m; q.bad = b; q.c = c;
        });
        mx = sh.bc.f; bad = sh.bc.bad; fin = sh.bc.c;
    }
    const int64_t t = a.tokens ? a.tokens[row] : -1;
    if (bad || fin == 0) {                                           // undefined row: NaN, ids -1, NaN
        if (rank == 0) {
            if (threadIdx.x == 0) a.lp[o] = NAN;
            for (int i = threadIdx.x; i < a.n_top; i += SP_THREADS) { a.ids[o * a.top_ld + i] = -1; a.top[o * a.top_ld + i] = NAN; }
        }
        cluster.sync();                                              // no CTA leaves while another may read its exchange slot
        return;
    }
    // 2. lse = m + log sum exp(x - m) over the finite entries, float64 (exp(-inf) is 0)
    double z = 0.0;
    for (int i = threadIdx.x; i < n; i += SP_THREADS) z += exp((double)s_row[i] - (double)mx);
    const double lse = (double)mx + log(cluster_sum_d(sh, ph, z));
    // 3. the chosen token: written by the CTA that holds it (rank 0 for a token outside the vocabulary)
    if (threadIdx.x == 0) {
        if (t >= 0 && t < a.vocab) {
            if (t >= lo && t < lo + n) a.lp[o] = (float)((double)s_row[t - lo] - lse);
        } else if (rank == 0) {
            a.lp[o] = NAN;
        }
    }
    if (a.n_top == 0) { cluster.sync(); return; }
    // 4. the top K = min(N, #finite): the key of rank K, then this CTA's entries at or above it
    const unsigned K = min((unsigned)a.n_top, fin);
    const unsigned long long thr = K == fin ? 0ull : radix_descent(sh, ph, LogitEval{}, s_row, n, lo, false, K, 0).key;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += SP_THREADS) {
        const float x = s_row[i];
        const unsigned long long key = logit_key(x, lo + i);
        if (isfinite(x) && key >= thr) {
            const unsigned q = atomicAdd(&s_cnt, 1u);                // the slot does not matter: ranks come from the keys
            s_key[q] = key; s_val[q] = x;
        }
    }
    cluster.sync();                                                  // every CTA's list is complete
    // 5. rank of each listed entry = listed keys above it, over the cluster; entries past #finite get -1 / -inf
    if (threadIdx.x < s_cnt) {
        const unsigned long long key = s_key[threadIdx.x];
        unsigned r = 0;
#pragma unroll
        for (int c = 0; c < SP_CL; c++) {
            const unsigned cnt = *cluster.map_shared_rank(&s_cnt, c);
            const unsigned long long* keys = cluster.map_shared_rank(&s_key[0], c);
            for (unsigned e = 0; e < cnt; e++) r += keys[e] > key ? 1u : 0u;
        }
        const int id = (SP_MAX_VOCAB - 1) - (int)(key & ((1u << SP_ID_BITS) - 1));
        a.ids[o * a.top_ld + r] = id;
        a.top[o * a.top_ld + r] = (float)((double)s_val[threadIdx.x] - lse);
    }
    if (rank == 0)
        for (int i = (int)K + threadIdx.x; i < a.n_top; i += SP_THREADS) { a.ids[o * a.top_ld + i] = -1; a.top[o * a.top_ld + i] = -INFINITY; }
    cluster.sync();                                                  // no CTA leaves while another may read its list
}

bool g_toplp_attr[EXL_MAX_DEVICES];

} // namespace

int exl_top_logprobs_launch(const float* logits, int rows, int vocab, int64_t logits_ld, const int64_t* tokens, int n_top,
                            const int* slot_host, const int* j_host, const int* status, int n_slots, int64_t out_ld, float* lp,
                            int64_t* top_ids, float* top_lp, int64_t top_ld, cudaStream_t stream)
{
    if (!logits || !lp)
        return exl_set_err(EXL_ERR_ARG, "top_logprobs: NULL pointer (logits %p, lp %p)", (const void*)logits, (void*)lp);
    if (rows < 1 || rows > EXL_RAGGED_MAX_SEQ)
        return exl_set_err(EXL_ERR_ARG, "top_logprobs: rows %d outside [1, %d]", rows, EXL_RAGGED_MAX_SEQ);
    if (vocab < 1 || vocab > SP_MAX_VOCAB) return exl_set_err(EXL_ERR_ARG, "top_logprobs: vocab %d outside [1, %d]", vocab, SP_MAX_VOCAB);
    if (logits_ld < vocab) return exl_set_err(EXL_ERR_ARG, "top_logprobs: logits_ld %lld < vocab %d", (long long)logits_ld, vocab);
    if (n_top < 0 || n_top > EXL_TOPLP_MAX) return exl_set_err(EXL_ERR_ARG, "top_logprobs: n_top %d outside [0, %d]", n_top, EXL_TOPLP_MAX);
    if (n_top > 0 && (!top_ids || !top_lp || top_ld < n_top))
        return exl_set_err(EXL_ERR_ARG, "top_logprobs: n_top %d with top_ids %p, top_lp %p, top_ld %lld", n_top, (void*)top_ids,
                           (void*)top_lp, (long long)top_ld);
    TopArgs a{};
    if (slot_host) {
        if (!j_host || !status)
            return exl_set_err(EXL_ERR_ARG, "top_logprobs: slot_host without j_host (%p) or status (%p)", (const void*)j_host,
                               (const void*)status);
        if (n_slots < 1 || n_slots > EXL_RAGGED_MAX_SEQ)
            return exl_set_err(EXL_ERR_ARG, "top_logprobs: n_slots %d outside [1, %d]", n_slots, EXL_RAGGED_MAX_SEQ);
        bool seen[EXL_RAGGED_MAX_SEQ] = {};
        for (int r = 0; r < rows; r++) {
            const int s = slot_host[r];
            if (s < -1 || s >= n_slots)
                return exl_set_err(EXL_ERR_ARG, "top_logprobs: row %d: slot %d outside [-1, n_slots %d)", r, s, n_slots);
            if (s >= 0) {
                if (seen[s]) return exl_set_err(EXL_ERR_ARG, "top_logprobs: row %d: slot %d named twice", r, s);
                seen[s] = true;
                if (j_host[r] < 0 || j_host[r] >= out_ld)
                    return exl_set_err(EXL_ERR_ARG, "top_logprobs: row %d: j %d outside [0, out_ld %lld)", r, j_host[r], (long long)out_ld);
            }
            a.slot[r] = s; a.j[r] = j_host[r];
        }
        a.status = status; a.out_ld = out_ld;
    }
    a.logits = logits; a.ld = logits_ld; a.vocab = vocab; a.slice = (vocab + SP_CL - 1) / SP_CL;
    a.tokens = tokens; a.n_top = n_top; a.top_ld = n_top > 0 ? top_ld : 0;
    a.lp = lp; a.ids = top_ids; a.top = top_lp;

    int dev = 0;
    EXL_CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= EXL_MAX_DEVICES) return exl_set_err(EXL_ERR_ARG, "top_logprobs: device %d", dev);
    if (!g_toplp_attr[dev]) {
        EXL_CUDA_TRY(cudaFuncSetAttribute(top_logprobs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SP_MAX_SLICE * (int)sizeof(float)));
        g_toplp_attr[dev] = true;
    }
    top_logprobs_kernel<<<dim3(SP_CL, rows), SP_THREADS, (size_t)a.slice * sizeof(float), stream>>>(a);
    EXL_CHECK_LAUNCH("top_logprobs_kernel");
    return EXL_OK;
}
