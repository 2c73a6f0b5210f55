// beam.cu -- beam search on the device: exl_beam_select (the best candidates across the beams' kept sets, or the first expansion's
// draw without replacement) and exl_kv_copy_rows (cache rows of one sequence copied to another, every layer, K and V, one launch).
//
// Select, expand mode   launch 1: one thread-block cluster of SP_CL CTAs per row (sample_kernel's layout, csrc/sample_select.cuh)
//                       keeps the row's slice in shared memory, checks it, counts its positive entries and finds the key of rank
//                       k = min(beams, #positive) with the sampler's radix descent over desc_key (probability descending, ties to
//                       the lower id); the tokens at or above that key -- the row's best k -- go to the work buffer.  Within a row
//                       the score score_host[r] + log((double)p) grows with p, so no other token of the row can be among the best.
//                       launch 2: one CTA loads every row's candidates, ranks each by counting the candidates before it under
//                       (score descending, row ascending, token ascending) and keeps ranks < min(beams, #candidates); the kept
//                       ones are laid out by (row ascending, score descending, token ascending).  Ranks come from integer counts
//                       over a total order, so the output does not depend on where launch 1 put a candidate.
// Select, first mode    launch 2 alone over the one row: up to `beams` successive inverse-CDF draws without replacement, thread t
//                       owning the contiguous run [t * per, (t + 1) * per) of the vocabulary, masses in the sampler's 2^-60 fixed
//                       point, integer scans only; the drawn tokens are returned sorted by id.
// Copy                  one CTA per (layer, K or V, KV head, pair): each is one contiguous run of (row_hi - row_lo) * head_dim
//                       halves, copied with 16-byte loads and stores, four in flight per thread.
#include "sample_select.cuh"
#include <cmath>

namespace {

constexpr int BS_MERGE_THREADS = 1024;

struct BeamTopArgs {
    const float* dist; int64_t ld; int vocab; int slice; int beams;
    float2* cand;                 // [rows][beams] (p, token id as int bits)
    int* n_cand;                  // [rows]: the row's candidates, -1 for an undefined row
};

struct BeamMergeArgs {
    const float* dist; int64_t ld; int vocab; int rows; int beams; int first;
    double score[EXL_RAGGED_MAX_SEQ];
    const float* u;
    const float2* cand; const int* n_cand;
    int* parent; int64_t* token; float* prob; double* out_score; int* count;
};

__device__ __forceinline__ bool bad_prob(float p) { return !(p >= 0.0f) || isinf(p); }     // NaN, negative or infinite

__global__ void __cluster_dims__(SP_CL, 1, 1) __launch_bounds__(SP_THREADS, 1) beam_topk_kernel(const __grid_constant__ BeamTopArgs a)
{
    extern __shared__ __align__(16) float s_row[];
    __shared__ Shared sh;
    __shared__ unsigned s_pos;
    cg::cluster_group cluster = cg::this_cluster();
    const int row = blockIdx.y;
    const int rank = (int)cluster.block_rank();
    const int lo = rank * a.slice;
    const int n = max(0, min(a.slice, a.vocab - lo));
    int ph = 0;

    const float* d = a.dist + (int64_t)row * a.ld + lo;
    int bad = 0;
    unsigned pos = 0;
    for (int i = threadIdx.x; i < n; i += SP_THREADS) {
        const float p = d[i];
        s_row[i] = p;
        bad |= bad_prob(p);
        pos += p > 0.0f ? 1u : 0u;
    }
    {
        Part p{}; p.c = block_sum_c(pos, sh); p.bad = block_or(bad, sh);
        cluster_exchange(sh, ph, p, [](const Part* ps, Part& o) {
            unsigned c = 0; int b = 0;
            for (int r = 0; r < SP_CL; r++) { c += ps[r].c; b |= ps[r].bad; }
            o.c = c; o.bad = b;
        });
    }
    const unsigned npos = sh.bc.c;
    if (sh.bc.bad || npos == 0) {
        if (rank == 0 && threadIdx.x == 0) a.n_cand[row] = -1;
        cluster.sync();                                              // no CTA leaves while another may read its exchange slot
        return;
    }
    const unsigned k = min((unsigned)a.beams, npos);
    const Row R;                                                     // no filter: every token is in, keyed by desc_key(p, id)
    const unsigned long long thr = radix_descent(sh, ph, R, s_row, n, lo, 1, false, k, 0).key;
    // this CTA's share of the best k goes after the shares of the lower ranks
    unsigned mine = 0;
    for (int i = threadIdx.x; i < n; i += SP_THREADS) mine += desc_key(s_row[i], lo + i) >= thr ? 1u : 0u;
    {
        Part p{}; p.c = block_sum_c(mine, sh);
        cluster_exchange(sh, ph, p, [rank](const Part* ps, Part& o) {
            unsigned c = 0;
            for (int r = 0; r < rank; r++) c += ps[r].c;
            o.c = c;
        });
    }
    if (threadIdx.x == 0) s_pos = sh.bc.c;
    __syncthreads();
    float2* out = a.cand + (int64_t)row * a.beams;
    for (int i = threadIdx.x; i < n; i += SP_THREADS)
        if (desc_key(s_row[i], lo + i) >= thr) out[atomicAdd(&s_pos, 1u)] = make_float2(s_row[i], __int_as_float(lo + i));
    if (rank == 0 && threadIdx.x == 0) a.n_cand[row] = (int)k;
    cluster.sync();                                                  // keep this CTA's exchange slot alive until every CTA has read it
}

// (score descending, row ascending, token ascending): candidate j before candidate i
__device__ __forceinline__ bool before(const double* sc, const int* par, const int* tok, int j, int i)
{
    if (sc[j] != sc[i]) return sc[j] > sc[i];
    if (par[j] != par[i]) return par[j] < par[i];
    return tok[j] < tok[i];
}
// (row ascending, score descending, token ascending): the layout of the kept candidates
__device__ __forceinline__ bool before_out(const double* sc, const int* par, const int* tok, int j, int i)
{
    if (par[j] != par[i]) return par[j] < par[i];
    if (sc[j] != sc[i]) return sc[j] > sc[i];
    return tok[j] < tok[i];
}

__global__ void __launch_bounds__(BS_MERGE_THREADS, 1) beam_merge_kernel(const __grid_constant__ BeamMergeArgs a)
{
    extern __shared__ __align__(16) unsigned char s_raw[];
    const int cap = a.first ? a.beams : a.rows * a.beams;
    double* sc = reinterpret_cast<double*>(s_raw);
    float* pr = reinterpret_cast<float*>(sc + cap);
    int* par = reinterpret_cast<int*>(pr + cap);
    int* tok = par + cap;
    int* top = tok + cap;                                            // [beams]: candidate index of rank r
    __shared__ int s_n;
    __shared__ unsigned long long s_m[BS_MERGE_THREADS / 32];
    __shared__ int s_l[BS_MERGE_THREADS / 32];
    __shared__ int s_pick;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    if (!a.first) {
        if (threadIdx.x == 0) {
            int n = 0;
            for (int r = 0; r < a.rows; r++) { if (a.n_cand[r] < 0) { n = -1; break; } n += a.n_cand[r]; }
            s_n = n;
        }
        __syncthreads();
        const int n = s_n;
        if (n < 0) {
            if (threadIdx.x == 0) *a.count = -1;
            for (int j = threadIdx.x; j < a.beams; j += BS_MERGE_THREADS) {
                a.parent[j] = -1; a.token[j] = -1; a.prob[j] = NAN; a.out_score[j] = NAN;
            }
            return;
        }
        for (int r = 0, off = 0; r < a.rows; off += a.n_cand[r], r++)
            for (int j = threadIdx.x; j < a.n_cand[r]; j += BS_MERGE_THREADS) {
                const float2 c = a.cand[(int64_t)r * a.beams + j];
                sc[off + j] = a.score[r] + log((double)c.x);
                pr[off + j] = c.x; par[off + j] = r; tok[off + j] = __float_as_int(c.y);
            }
        const int K = min(a.beams, n);
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += BS_MERGE_THREADS) {
            int c = 0;
            for (int j = 0; j < n && c < K; j++) c += before(sc, par, tok, j, i) ? 1 : 0;
            if (c < K) top[c] = i;
        }
        __syncthreads();
        for (int t = threadIdx.x; t < K; t += BS_MERGE_THREADS) {
            const int i = top[t];
            int o = 0;
            for (int s = 0; s < K; s++) o += before_out(sc, par, tok, top[s], i) ? 1 : 0;
            a.parent[o] = par[i]; a.token[o] = tok[i]; a.prob[o] = pr[i]; a.out_score[o] = sc[i];
        }
        for (int j = K + threadIdx.x; j < a.beams; j += BS_MERGE_THREADS) {
            a.parent[j] = -1; a.token[j] = -1; a.prob[j] = NAN; a.out_score[j] = NAN;
        }
        if (threadIdx.x == 0) *a.count = K;
        return;
    }

    // first mode: one row, draws without replacement
    const float* d = a.dist;
    const int per = (a.vocab + BS_MERGE_THREADS - 1) / BS_MERGE_THREADS;
    const int i0 = min(a.vocab, (int)threadIdx.x * per), i1 = min(a.vocab, i0 + per);
    unsigned long long run = 0;
    int bad = 0, npos = 0;
    for (int i = i0; i < i1; i++) {
        const float p = d[i];
        bad |= bad_prob(p);
        npos += p > 0.0f;
        run += fix60(p);
    }
    bad = __any_sync(0xffffffffu, bad);
    npos = __reduce_add_sync(0xffffffffu, (unsigned)npos);
    if (lane == 0) { s_l[warp] = bad; s_m[warp] = (unsigned long long)npos; }
    __syncthreads();
    if (threadIdx.x == 0) {
        int b = 0; unsigned long long c = 0;
        for (int w = 0; w < BS_MERGE_THREADS / 32; w++) { b |= s_l[w]; c += s_m[w]; }
        s_n = b ? -1 : (int)c;
    }
    __syncthreads();
    if (s_n <= 0) {
        if (threadIdx.x == 0) *a.count = -1;
        for (int j = threadIdx.x; j < a.beams; j += BS_MERGE_THREADS) {
            a.parent[j] = -1; a.token[j] = -1; a.prob[j] = NAN; a.out_score[j] = NAN;
        }
        return;
    }
    const int K = min(a.beams, s_n);
    for (int j = 0; j < K; j++) {
        // this run's remaining mass: its full mass less the tokens drawn from it
        unsigned long long mine = run;
        for (int s = 0; s < j; s++) if (tok[s] >= i0 && tok[s] < i1) mine -= fix60(pr[s]);
        unsigned long long incl = mine;
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
        __syncthreads();
        if (lane == 31) s_m[warp] = incl;
        if (threadIdx.x == 0) s_pick = -1;
        __syncthreads();
        unsigned long long base = incl - mine, total = 0;
        for (int w = 0; w < BS_MERGE_THREADS / 32; w++) { if (w < warp) base += s_m[w]; total += s_m[w]; }
        auto drawn = [&](int i) { for (int s = 0; s < j; s++) if (tok[s] == i) return true; return false; };
        const unsigned long long U = (unsigned long long)((double)a.u[j] * (double)total);
        if (U < total) {
            if (base <= U && U < base + mine) {
                unsigned long long cum = base;
                for (int i = i0; i < i1; i++) {
                    if (drawn(i)) continue;
                    cum += fix60(d[i]);
                    if (cum > U) { s_pick = i; break; }
                }
            }
        }
        __syncthreads();
        if (s_pick < 0) {                                            // rounding left u at or above the total: the largest remaining positive id
            int last = -1;
            for (int i = i1 - 1; i >= i0; i--) if (d[i] > 0.0f && !drawn(i)) { last = i; break; }
            for (int o = 16; o; o >>= 1) last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
            __syncthreads();
            if (lane == 0) s_l[warp] = last;
            __syncthreads();
            if (threadIdx.x == 0) { int m = -1; for (int w = 0; w < BS_MERGE_THREADS / 32; w++) m = max(m, s_l[w]); s_pick = m; }
            __syncthreads();
        }
        if (threadIdx.x == 0) { tok[j] = s_pick; pr[j] = d[s_pick]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        for (int j = 0; j < K; j++) {                                // sorted by id (K <= 64: insertion into place)
            int o = 0;
            for (int s = 0; s < K; s++) o += tok[s] < tok[j];
            a.parent[o] = 0; a.token[o] = tok[j]; a.prob[o] = pr[j]; a.out_score[o] = a.score[0] + log((double)pr[j]);
        }
        for (int j = K; j < a.beams; j++) { a.parent[j] = -1; a.token[j] = -1; a.prob[j] = NAN; a.out_score[j] = NAN; }
        *a.count = K;
    }
}

// ---- exl_kv_copy_rows ---------------------------------------------------------------------------------------------------------
constexpr int KC_THREADS = 256;
constexpr int KC_UNROLL = 4;

struct KvCopyArgs {
    half* cache[2 * EXL_KV_COPY_MAX_LAYERS];   // layer l: K at 2 l, V at 2 l + 1
    exl_kv_copy_pair pair[EXL_RAGGED_MAX_SEQ];
    int n_pairs, kv_heads, max_seq, head_dim;
};

__global__ void __launch_bounds__(KC_THREADS) kv_copy_rows_kernel(const __grid_constant__ KvCopyArgs a)
{
    unsigned u = blockIdx.x;
    const int pi = (int)(u % (unsigned)a.n_pairs); u /= (unsigned)a.n_pairs;
    const int h = (int)(u % (unsigned)a.kv_heads); u /= (unsigned)a.kv_heads;
    const exl_kv_copy_pair p = a.pair[pi];
    half* base = a.cache[u];
    const int64_t vecs = (int64_t)(p.row_hi - p.row_lo) * a.head_dim / 8;
    const uint4* src = reinterpret_cast<const uint4*>(base + (((int64_t)p.src * a.kv_heads + h) * a.max_seq + p.row_lo) * a.head_dim);
    uint4* dst = reinterpret_cast<uint4*>(base + (((int64_t)p.dst * a.kv_heads + h) * a.max_seq + p.row_lo) * a.head_dim);
    int64_t i = threadIdx.x;
    for (; i + (KC_UNROLL - 1) * KC_THREADS < vecs; i += KC_UNROLL * KC_THREADS) {
        uint4 v[KC_UNROLL];
#pragma unroll
        for (int r = 0; r < KC_UNROLL; r++) v[r] = __ldcs(src + i + r * KC_THREADS);
#pragma unroll
        for (int r = 0; r < KC_UNROLL; r++) dst[i + r * KC_THREADS] = v[r];
    }
    for (; i < vecs; i += KC_THREADS) dst[i] = __ldcs(src + i);
}

bool g_topk_attr[EXL_MAX_DEVICES];

} // namespace

int exl_beam_select_launch(const float* dist, int rows, int vocab, int64_t dist_ld, const double* score_host, int beams, int mode,
                           const float* u, void* work, int64_t work_bytes, int* parent, int64_t* token, float* prob, double* score,
                           int* count, cudaStream_t stream)
{
    if (!dist || !score_host || !work || !parent || !token || !prob || !score || !count)
        return exl_set_err(EXL_ERR_ARG, "beam_select: NULL pointer (dist %p, score_host %p, work %p, parent %p, token %p, prob %p, "
                           "score %p, count %p)", (const void*)dist, (const void*)score_host, work, (void*)parent, (void*)token,
                           (void*)prob, (void*)score, (void*)count);
    if (mode != EXL_BEAM_EXPAND && mode != EXL_BEAM_FIRST)
        return exl_set_err(EXL_ERR_ARG, "beam_select: mode %d is neither EXL_BEAM_EXPAND (0) nor EXL_BEAM_FIRST (1)", mode);
    if (rows < 1 || rows > EXL_RAGGED_MAX_SEQ) return exl_set_err(EXL_ERR_ARG, "beam_select: rows %d outside [1, %d]", rows, EXL_RAGGED_MAX_SEQ);
    if (mode == EXL_BEAM_FIRST && rows != 1) return exl_set_err(EXL_ERR_ARG, "beam_select: rows %d in first mode (one row)", rows);
    if (mode == EXL_BEAM_FIRST && !u) return exl_set_err(EXL_ERR_ARG, "beam_select: u is NULL in first mode");
    if (beams < 1 || beams > EXL_RAGGED_MAX_SEQ) return exl_set_err(EXL_ERR_ARG, "beam_select: beams %d outside [1, %d]", beams, EXL_RAGGED_MAX_SEQ);
    if (vocab < 1 || vocab > SP_MAX_VOCAB) return exl_set_err(EXL_ERR_ARG, "beam_select: vocab %d outside [1, %d]", vocab, SP_MAX_VOCAB);
    if (dist_ld < vocab) return exl_set_err(EXL_ERR_ARG, "beam_select: dist_ld %lld < vocab %d", (long long)dist_ld, vocab);
    if (work_bytes < EXL_BEAM_WORK_BYTES(rows, beams))
        return exl_set_err(EXL_ERR_ARG, "beam_select: work_bytes %lld < EXL_BEAM_WORK_BYTES(%d, %d) = %lld", (long long)work_bytes, rows,
                           beams, (long long)EXL_BEAM_WORK_BYTES(rows, beams));
    if (reinterpret_cast<uintptr_t>(work) % 16) return exl_set_err(EXL_ERR_ARG, "beam_select: work %p is not 16-byte aligned", work);
    BeamMergeArgs m{};
    for (int r = 0; r < rows; r++) {
        if (std::isnan(score_host[r]) || score_host[r] == INFINITY)
            return exl_set_err(EXL_ERR_ARG, "beam_select: score_host[%d] %g is NaN or +inf", r, score_host[r]);
        m.score[r] = score_host[r];
    }
    int dev = 0;
    EXL_CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= EXL_MAX_DEVICES) return exl_set_err(EXL_ERR_ARG, "beam_select: device %d", dev);
    if (!g_topk_attr[dev]) {
        EXL_CUDA_TRY(cudaFuncSetAttribute(beam_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SP_MAX_SLICE * (int)sizeof(float)));
        const int merge_max = EXL_RAGGED_MAX_SEQ * EXL_RAGGED_MAX_SEQ * (8 + 4 + 4 + 4) + EXL_RAGGED_MAX_SEQ * 4;
        EXL_CUDA_TRY(cudaFuncSetAttribute(beam_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, merge_max));
        g_topk_attr[dev] = true;
    }
    float2* cand = reinterpret_cast<float2*>(work);
    int* n_cand = reinterpret_cast<int*>(cand + (int64_t)rows * beams);
    if (mode == EXL_BEAM_EXPAND) {
        BeamTopArgs t{dist, dist_ld, vocab, (vocab + SP_CL - 1) / SP_CL, beams, cand, n_cand};
        beam_topk_kernel<<<dim3(SP_CL, rows), SP_THREADS, (size_t)t.slice * sizeof(float), stream>>>(t);
        EXL_CHECK_LAUNCH("beam_topk_kernel");
    }
    m.dist = dist; m.ld = dist_ld; m.vocab = vocab; m.rows = rows; m.beams = beams; m.first = mode == EXL_BEAM_FIRST;
    m.u = u; m.cand = cand; m.n_cand = n_cand;
    m.parent = parent; m.token = token; m.prob = prob; m.out_score = score; m.count = count;
    const int cap = m.first ? beams : rows * beams;
    const size_t smem = (size_t)cap * (8 + 4 + 4 + 4) + (size_t)beams * 4;
    beam_merge_kernel<<<1, BS_MERGE_THREADS, smem, stream>>>(m);
    EXL_CHECK_LAUNCH("beam_merge_kernel");
    return EXL_OK;
}

int exl_kv_copy_rows_launch(void* const* k_caches, void* const* v_caches, int n_layers, int num_cache_seqs, int num_kv_heads,
                            int max_seq_len, int head_dim, const exl_kv_copy_pair* pairs, int n_pairs, cudaStream_t stream)
{
    if (!k_caches || !v_caches || !pairs)
        return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: NULL pointer (k_caches %p, v_caches %p, pairs %p)", (const void*)k_caches,
                           (const void*)v_caches, (const void*)pairs);
    if (n_layers < 1 || n_layers > EXL_KV_COPY_MAX_LAYERS)
        return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: n_layers %d outside [1, %d]", n_layers, EXL_KV_COPY_MAX_LAYERS);
    if (n_pairs < 1 || n_pairs > EXL_RAGGED_MAX_SEQ)
        return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: n_pairs %d outside [1, %d]", n_pairs, EXL_RAGGED_MAX_SEQ);
    if (num_cache_seqs < 2) return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: num_cache_seqs %d < 2", num_cache_seqs);
    if (num_kv_heads < 1) return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: num_kv_heads %d < 1", num_kv_heads);
    if (max_seq_len < 1) return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: max_seq_len %d < 1", max_seq_len);
    if (head_dim < 8 || head_dim % 8) return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: head_dim %d is not a positive multiple of 8", head_dim);
    if ((int64_t)num_cache_seqs * num_kv_heads * max_seq_len * head_dim > ((int64_t)1 << 40))
        return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: cache of %d x %d x %d x %d halves", num_cache_seqs, num_kv_heads, max_seq_len, head_dim);
    KvCopyArgs a{};
    for (int l = 0; l < n_layers; l++) {
        for (int kv = 0; kv < 2; kv++) {
            void* c = (kv ? v_caches : k_caches)[l];
            if (!c || reinterpret_cast<uintptr_t>(c) % 16)
                return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: %s cache of layer %d (%p) is NULL or not 16-byte aligned", kv ? "V" : "K", l, c);
            a.cache[2 * l + kv] = reinterpret_cast<half*>(c);
        }
    }
    for (int i = 0; i < n_pairs; i++) {
        const exl_kv_copy_pair p = pairs[i];
        if (p.src < 0 || p.src >= num_cache_seqs || p.dst < 0 || p.dst >= num_cache_seqs)
            return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: pair %d copies sequence %d to %d; the caches hold [0, %d)", i, p.src, p.dst,
                               num_cache_seqs);
        if (p.row_lo < 0 || p.row_lo > p.row_hi || p.row_hi > max_seq_len)
            return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: pair %d rows [%d, %d) outside [0, max_seq_len %d]", i, p.row_lo, p.row_hi,
                               max_seq_len);
        for (int j = 0; j < n_pairs; j++) {
            if (pairs[j].dst == p.src)
                return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: sequence %d is the source of pair %d and the destination of pair %d", p.src, i, j);
            if (j < i && pairs[j].dst == p.dst)
                return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: sequence %d is the destination of pairs %d and %d", p.dst, j, i);
        }
        a.pair[i] = p;
    }
    a.n_pairs = n_pairs; a.kv_heads = num_kv_heads; a.max_seq = max_seq_len; a.head_dim = head_dim;
    const long long blocks = 2LL * n_layers * num_kv_heads * n_pairs;
    if (blocks > 0x7fffffffLL) return exl_set_err(EXL_ERR_ARG, "kv_copy_rows: %lld blocks", blocks);
    kv_copy_rows_kernel<<<(unsigned)blocks, KC_THREADS, 0, stream>>>(a);
    EXL_CHECK_LAUNCH("kv_copy_rows_kernel");
    return EXL_OK;
}
