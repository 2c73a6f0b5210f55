// sample.cu -- exl_sample: the generator's token sampling (generator.py:91-170 with apply_rep_penalty_cpu and the bos logit of
// gen_single_token) on the device, one launch for up to EXL_RAGGED_MAX_SEQ rows.
//
// Layout     one thread-block cluster of SP_CL CTAs per row.  CTA r owns the contiguous slice [r * slice, (r + 1) * slice) of the
//            vocabulary (slice = ceil(vocab / SP_CL) <= 32768) and keeps it in shared memory for the whole call, so every pass
//            after the first reads shared memory, whatever the vocabulary size.  Cluster-wide quantities (the row maximum, sums,
//            histograms) are merged over distributed shared memory; every CTA reads the same merged values in the same order and
//            so takes the same decisions.
// Penalty    the history window is scanned once: integer atomicMin of the position (newest first) per token of the slice, in the
//            slice buffer itself, gives each token its newest occurrence; v at that position comes from the fp32 recurrence
//            v += dv computed step by step (bit-exact with exl_apply_rep_penalty).
// Filters    top-k, top-p and typical each keep a prefix of an order: probability descending (top-k, top-p) or entropy deviation
//            ascending (typical), ties to the lower token id.  Both orders are 50-bit keys (the float's bits above the inverted
//            token id, so keys are unique), and each cut is found by a radix descent over the key in five 10-bit digits with
//            bucket histograms of counts and of probability mass -- no sort.  Mass is summed in 2^-60 fixed point with integer
//            atomics, so its order does not matter; fp32 sums (softmax, normalisations) use one fixed reduction order.  Two
//            launches are bitwise equal.
// Draw       inverse CDF in ascending token-id order over the kept set, in the same fixed point.
#include "sample_select.cuh"
#include <cmath>
#include <cstdio>

namespace {

// One row's settings: exl_sample_params without its padding.  exl_sample gives every row the same; exl_sample_rows its own.
struct RowParams {
    float temperature; int top_k; float top_p, min_p, typical;
    float pmax; int sustain, decay, bos, n_banned;
    const int* banned;
};

struct SampleArgs {
    const float* logits; int64_t ld; int vocab; int slice;
    const int64_t* hist; int64_t hist_ld; int hist_len[EXL_RAGGED_MAX_SEQ];
    const int64_t* tail; int tail_at;            // history positions >= tail_at read tail[pos - tail_at] (tail NULL: none)
    const float* u; int64_t* tokens; float* probs; float* dist;
    RowParams rp[EXL_RAGGED_MAX_SEQ];            // a cluster is one row, so every branch on a row's settings is uniform in it
};
static_assert(sizeof(RowParams) == 48, "RowParams layout");
static_assert(sizeof(SampleArgs) <= 4096, "SampleArgs must fit the classic 4 KB kernel parameter space");

__global__ void __cluster_dims__(SP_CL, 1, 1) __launch_bounds__(SP_THREADS, 1) sample_kernel(const __grid_constant__ SampleArgs a)
{
    extern __shared__ __align__(16) float s_row[];
    __shared__ Shared sh;
    int* s_int = reinterpret_cast<int*>(s_row);
    cg::cluster_group cluster = cg::this_cluster();
    const int row = blockIdx.y;
    const int rank = (int)cluster.block_rank();
    const int lo = rank * a.slice;
    const int n = max(0, min(a.slice, a.vocab - lo));
    int ph = 0;
    int bad = 0;
    const RowParams& rs = a.rp[row];

    // 1. repetition penalty: newest window position of each token of the slice
    const bool pen = a.hist != nullptr && rs.pmax != 1.0f && a.hist_len[row] > 0;
    long long s0 = 0;
    const float dv = rs.decay ? (1.0f - rs.pmax) / (float)rs.decay : 0.0f;
    if (pen)
        s0 = penalty_scan(sh, s_int, a.hist + (int64_t)row * a.hist_ld, a.tail, a.tail_at, a.hist_len[row], rs.pmax, rs.sustain, rs.decay,
                          dv, a.vocab, lo, n, bad);
    // 2. penalised logits, bos, banned
    const float* lg = a.logits + (int64_t)row * a.ld + lo;
    for (int i = threadIdx.x; i < n; i += SP_THREADS) {
        float x = lg[i];
        if (pen) x = penalise(sh, x, s_int[i], s0, dv);
        if (lo + i == rs.bos) x = -10000.0f;
        s_row[i] = x;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < rs.n_banned; k += SP_THREADS) {
        const int t = rs.banned[k];
        if (t < 0 || t >= a.vocab) { bad = 1; continue; }
        if (t >= lo && t < lo + n) s_row[t - lo] = -INFINITY;
    }
    __syncthreads();
    // 3. temperature, + 1e-8, softmax
    float mx = -INFINITY;
    for (int i = threadIdx.x; i < n; i += SP_THREADS) {
        const float y = __fadd_rn(__fdiv_rn(s_row[i], rs.temperature), 1e-8f);
        s_row[i] = y;
        if (isnan(y)) bad = 1;
        mx = fmaxf(mx, y);
    }
    {
        Part p{}; p.f = block_max_f(mx, sh); p.bad = block_or(bad, sh);
        cluster_exchange(sh, ph, p, [](const Part* ps, Part& o) {
            float m = -INFINITY; int b = 0;
            for (int r = 0; r < SP_CL; r++) { m = fmaxf(m, ps[r].f); b |= ps[r].bad; }
            o.f = m; o.bad = b;
        });
        mx = sh.bc.f; bad = sh.bc.bad;
    }
    if (bad || mx == -INFINITY) {                                    // undefined row: -1 / NaN
        if (rank == 0 && threadIdx.x == 0) { a.tokens[row] = -1; a.probs[row] = NAN; }
        if (a.dist) for (int i = threadIdx.x; i < n; i += SP_THREADS) a.dist[(int64_t)row * a.vocab + lo + i] = NAN;
        cluster.sync();                                              // no CTA leaves while another may read its exchange slot
        return;
    }
    float z = 0.f;
    for (int i = threadIdx.x; i < n; i += SP_THREADS) { const float e = expf(s_row[i] - mx); s_row[i] = e; z += e; }
    z = cluster_sum_f(sh, ph, z);
    for (int i = threadIdx.x; i < n; i += SP_THREADS) s_row[i] = s_row[i] / z;
    __syncthreads();

    Row R;
    unsigned len = (unsigned)a.vocab;                                // length of the ordered list at the current stage
    // 4. top-k, then L1 normalisation
    if (rs.top_k > 0) {
        R.kk = radix_descent(sh, ph, ProbEval{R, 1}, s_row, n, lo, false, (unsigned)rs.top_k, 0).key;
        len = (unsigned)rs.top_k;
        float s = 0.f;
        for (int i = threadIdx.x; i < n; i += SP_THREADS) if (desc_key(s_row[i], lo + i) >= R.kk) s += s_row[i];
        R.sk = fmaxf(cluster_sum_f(sh, ph, s), 1e-12f);
    }
    // 5. top-p with its min_p test, then renormalise
    if (rs.top_p > 0.0f) {
        const unsigned long long T = (unsigned long long)((double)fminf(rs.top_p, 2.0f) * SP_FIX);
        const Descent c = radix_descent(sh, ph, ProbEval{R, 1}, s_row, n, lo, true, 0, T);
        const unsigned n_p = c.found ? c.before : len;
        unsigned cm = 0;
        for (int i = threadIdx.x; i < n; i += SP_THREADS) {
            const Tok t = eval(R, s_row[i], lo + i, 1);
            cm += (t.in && t.w >= rs.min_p) ? 1u : 0u;
        }
        cm = cluster_sum_c(sh, ph, cm);
        const unsigned keep = max(1u, min(min(n_p, cm), len));
        if (c.found && keep == n_p) R.kp = c.key + 1;                // everything before the first token past top_p
        else if (keep == len) R.kp = 0;
        else R.kp = radix_descent(sh, ph, ProbEval{R, 1}, s_row, n, lo, false, keep, 0).key;
        len = keep;
        float s = 0.f;
        for (int i = threadIdx.x; i < n; i += SP_THREADS) {
            const Tok t = eval(R, s_row[i], lo + i, 2);
            if (t.in) s += t.w;
        }
        R.sp = fmaxf(cluster_sum_f(sh, ph, s), 1e-12f);
    }
    // 6. typical: order by |sum p log(p + eps) - log(p + eps)| ascending, the same prefix rule without min_p, renormalise
    if (rs.typical > 0.0f) {
        float s = 0.f;
        for (int i = threadIdx.x; i < n; i += SP_THREADS) {
            const Tok t = eval(R, s_row[i], lo + i, 2);
            if (t.in) s += t.w * logf(t.w + 1e-10f);
        }
        R.negent = cluster_sum_f(sh, ph, s);
        const unsigned long long T = (unsigned long long)((double)fminf(rs.typical, 2.0f) * SP_FIX);
        const Descent c = radix_descent(sh, ph, ProbEval{R, 3}, s_row, n, lo, true, 0, T);
        const unsigned n_t = c.found ? c.before : len;
        const unsigned keep = max(1u, min(n_t, len));
        if (c.found && keep == n_t) R.kt = c.key + 1;
        else if (keep == len) R.kt = 0;
        else R.kt = radix_descent(sh, ph, ProbEval{R, 3}, s_row, n, lo, false, keep, 0).key;
        float s2 = 0.f;
        for (int i = threadIdx.x; i < n; i += SP_THREADS) {
            const Tok t = eval(R, s_row[i], lo + i, 3);
            if (t.in) s2 += t.w;
        }
        R.st = fmaxf(cluster_sum_f(sh, ph, s2), 1e-12f);
    }
    const int level = rs.typical > 0.0f ? 3 : (rs.top_p > 0.0f ? 2 : 1);

    // 7. final distribution and the draw: thread t owns the contiguous run [t * per, (t + 1) * per) of the slice
    const int per = (n + SP_THREADS - 1) / SP_THREADS;
    const int i0 = min(n, (int)threadIdx.x * per), i1 = min(n, i0 + per);
    unsigned long long mine = 0;
    int last_kept = -1;
    for (int i = i0; i < i1; i++) {
        const Tok t = eval(R, s_row[i], lo + i, level);
        const float f = t.in ? t.w : 0.0f;
        if (a.dist) a.dist[(int64_t)row * a.vocab + lo + i] = f;
        if (t.in) { mine += fix60(f); last_kept = lo + i; }
    }
    // exclusive scan of the runs' masses inside the CTA
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long incl = mine;
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    int lk = last_kept;
    for (int o = 16; o; o >>= 1) lk = max(lk, __shfl_xor_sync(0xffffffffu, lk, o));
    __syncthreads();
    if (lane == 31) sh.redm[warp] = incl;
    if (lane == 0) sh.redi[warp] = lk;
    __syncthreads();
    unsigned long long base = incl - mine, cta_total = 0;
    int cta_last = -1;
    for (int w = 0; w < SP_THREADS / 32; w++) {
        if (w < warp) base += sh.redm[w];
        cta_total += sh.redm[w];
        cta_last = max(cta_last, sh.redi[w]);
    }
    Part p{}; p.m = cta_total; p.bad = cta_last;
    if (threadIdx.x == 0) sh.xch[ph & 1] = p;
    cluster.sync();
    unsigned long long before_cta = 0, total = 0;
    int row_last = -1;
    for (int r = 0; r < SP_CL; r++) {
        const Part q = *cluster.map_shared_rank(&sh.xch[ph & 1], r);
        if (r < rank) before_cta += q.m;
        total += q.m;
        row_last = max(row_last, q.bad);
    }
    const unsigned long long U = (unsigned long long)((double)a.u[row] * SP_FIX);
    if (U >= total) {                                                // rounding left u at or above the total: the largest kept id
        if (lo <= row_last && row_last < lo + n && row_last == last_kept) {
            a.tokens[row] = row_last;
            a.probs[row] = eval(R, s_row[row_last - lo], row_last, level).w;
        }
    } else {
        unsigned long long cum = before_cta + base;
        if (cum <= U && U < cum + mine) {
            for (int i = i0; i < i1; i++) {
                const Tok t = eval(R, s_row[i], lo + i, level);
                if (!t.in) continue;
                cum += fix60(t.w);
                if (cum > U) { a.tokens[row] = lo + i; a.probs[row] = t.w; break; }
            }
        }
    }
    cluster.sync();                                                  // keep this CTA's exchange slot alive until every CTA has read it
}

// ---- speculative verification (exl_spec_verify): the acceptance walk and the residual draw --------------------------------------
constexpr int SV_THREADS = 512;

struct VerifyArgs {
    const float* p;              // [k + 1][vocab]: sample_kernel's final distributions of the target rows
    const float* q; int64_t q_ld;
    const int64_t* drafts; const float* u;
    int k, vocab;
    int* n_acc; int64_t* tokens; float* probs;    // tokens / probs hold sample_kernel's draws of the target rows on entry
};

// One CTA.  Thread 0 walks the drafts (u_{j-1} q_j(d_j) < p_{j-1}(d_j) accepts d_j); after a rejection the block draws the
// correction from max(0, p_{j-1} - q_j) -- from p_{j-1} if rounding left that empty -- with u_k: thread t owns the contiguous
// run [t * per, (t + 1) * per) of the vocabulary, masses in the sampler's 2^-60 fixed point, integer scans only.
__global__ void __launch_bounds__(SV_THREADS, 1) spec_residual_kernel(const __grid_constant__ VerifyArgs a)
{
    __shared__ int s_acc, s_state, s_pick;
    __shared__ int64_t s_bonus; __shared__ float s_bonus_p;
    __shared__ unsigned long long s_m[SV_THREADS / 32];
    __shared__ int s_l[SV_THREADS / 32];
    if (threadIdx.x == 0) {
        int n = 0, state = 0;                                        // 0: all accepted, 1: d_{n+1} rejected, -1: undefined
        for (; n < a.k; n++) {
            if (a.tokens[n] < 0) { state = -1; break; }              // p_n undefined
            const int64_t d = a.drafts[n];
            if (d < 0 || d >= a.vocab) { state = -1; break; }
            const float qd = a.q[(int64_t)n * a.q_ld + d];
            if (!(qd > 0.0f) || !isfinite(qd)) { state = -1; break; }
            if (!(__fmul_rn(a.u[n], qd) < a.p[(int64_t)n * a.vocab + d])) { state = 1; break; }
        }
        if (state == 0 && a.tokens[a.k] < 0) state = -1;
        s_acc = n; s_state = state; s_pick = -1;
        s_bonus = a.tokens[a.k]; s_bonus_p = a.probs[a.k];
    }
    __syncthreads();
    const int n = s_acc;
    int state = s_state;
    if (state == 1) {
        const float* p = a.p + (int64_t)n * a.vocab;
        const float* q = a.q + (int64_t)n * a.q_ld;
        const int per = (a.vocab + SV_THREADS - 1) / SV_THREADS;
        const int i0 = min(a.vocab, (int)threadIdx.x * per), i1 = min(a.vocab, i0 + per);
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (int resid = 1; resid >= 0; resid--) {                   // the same decision in every thread: total is block-wide
            auto mass = [&](int i) { return fix60(resid ? fmaxf(p[i] - q[i], 0.0f) : p[i]); };
            unsigned long long mine = 0;
            int last = -1;
            for (int i = i0; i < i1; i++) { const unsigned long long m = mass(i); mine += m; if (m) last = i; }
            unsigned long long incl = mine;
            for (int o = 1; o < 32; o <<= 1) { const unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
            int lk = last;
            for (int o = 16; o; o >>= 1) lk = max(lk, __shfl_xor_sync(0xffffffffu, lk, o));
            __syncthreads();
            if (lane == 31) s_m[warp] = incl;
            if (lane == 0) s_l[warp] = lk;
            __syncthreads();
            unsigned long long base = incl - mine, total = 0;
            int row_last = -1;
            for (int w = 0; w < SV_THREADS / 32; w++) {
                if (w < warp) base += s_m[w];
                total += s_m[w];
                row_last = max(row_last, s_l[w]);
            }
            if (total == 0) continue;                                // only rounding empties the residual: draw from p_n
            const unsigned long long U = (unsigned long long)((double)a.u[a.k] * (double)total);
            if (U >= total) {                                        // rounding left u at or above the total: the largest id with mass
                if (threadIdx.x == 0) s_pick = row_last;
            } else if (base <= U && U < base + mine) {
                unsigned long long cum = base;
                for (int i = i0; i < i1; i++) {
                    cum += mass(i);
                    if (cum > U) { s_pick = i; break; }
                }
            }
            break;
        }
        __syncthreads();
        if (s_pick < 0) state = -1;                                  // no mass at all: a defined p row always has some
    }
    if (threadIdx.x == 0) {
        const int emitted = state < 0 ? 0 : n + 1;                   // tokens written before the -1 tail
        for (int j = 0; j <= a.k; j++) {
            int64_t t = -1; float pr = NAN;
            if (j < emitted) {
                if (j < n) t = a.drafts[j];
                else t = state == 0 ? s_bonus : (int64_t)s_pick;
                pr = j < n || state == 1 ? a.p[(int64_t)j * a.vocab + t] : s_bonus_p;
            }
            a.tokens[j] = t; a.probs[j] = pr;
        }
        *a.n_acc = state < 0 ? -1 : n;
    }
}

bool g_sample_attr[EXL_MAX_DEVICES];

} // namespace

// Checks one parameter set the way exl_sample always has; who is "sample" or "sample: row <b>" (exl_sample_rows names the row).
static int check_params(const exl_sample_params* p, int vocab, const char* who)
{
    if (!std::isfinite(p->temperature) || !(p->temperature > 0.0f))
        return exl_set_err(EXL_ERR_ARG, "%s: temperature %g is not finite and positive", who, (double)p->temperature);
    if (p->top_k < 0 || p->top_k > vocab) return exl_set_err(EXL_ERR_ARG, "%s: top_k %d outside [0, vocab %d]", who, p->top_k, vocab);
    if (!(p->top_p >= 0.0f)) return exl_set_err(EXL_ERR_ARG, "%s: top_p %g is negative", who, (double)p->top_p);
    if (!(p->min_p >= 0.0f)) return exl_set_err(EXL_ERR_ARG, "%s: min_p %g is negative", who, (double)p->min_p);
    if (!(p->typical >= 0.0f)) return exl_set_err(EXL_ERR_ARG, "%s: typical %g is negative", who, (double)p->typical);
    if (p->rep_sustain < -1) return exl_set_err(EXL_ERR_ARG, "%s: rep_sustain %d < -1", who, p->rep_sustain);
    if (p->rep_decay < 0) return exl_set_err(EXL_ERR_ARG, "%s: rep_decay %d < 0", who, p->rep_decay);
    if (p->n_banned < 0 || (p->n_banned > 0 && !p->banned))
        return exl_set_err(EXL_ERR_ARG, "%s: n_banned %d with banned %p", who, p->n_banned, (const void*)p->banned);
    return EXL_OK;
}

// per_row: row b uses p[b] (exl_sample_rows); else every row uses p[0]
static int sample_launch(const float* logits, int bsz, int vocab, int64_t logits_ld, const int64_t* history, int64_t hist_ld,
                         const int* hist_len, const exl_sample_params* p, bool per_row, const float* u, int64_t* tokens, float* probs,
                         float* dist, cudaStream_t stream, const int64_t* tail)
{
    if (!p) return exl_set_err(EXL_ERR_ARG, per_row ? "sample: p_rows is NULL" : "sample: params is NULL");
    if (!logits || !u || !tokens || !probs)
        return exl_set_err(EXL_ERR_ARG, "sample: NULL pointer (logits %p, u %p, tokens %p, probs %p)", (const void*)logits,
                           (const void*)u, (void*)tokens, (void*)probs);
    if (bsz < 1 || bsz > EXL_RAGGED_MAX_SEQ) return exl_set_err(EXL_ERR_ARG, "sample: bsz %d outside [1, %d]", bsz, EXL_RAGGED_MAX_SEQ);
    if (vocab < 1 || vocab > SP_MAX_VOCAB) return exl_set_err(EXL_ERR_ARG, "sample: vocab %d outside [1, %d]", vocab, SP_MAX_VOCAB);
    if (logits_ld < vocab) return exl_set_err(EXL_ERR_ARG, "sample: logits_ld %lld < vocab %d", (long long)logits_ld, vocab);
    for (int b = 0; b < (per_row ? bsz : 1); b++) {
        char who[32];
        if (per_row) snprintf(who, sizeof who, "sample: row %d", b);
        else snprintf(who, sizeof who, "sample");
        const int rc = check_params(p + b, vocab, who);
        if (rc != EXL_OK) return rc;
    }
    SampleArgs a{};
    if (history) {
        if (!hist_len) return exl_set_err(EXL_ERR_ARG, "sample: history without hist_len_host");
        for (int b = 0; b < (tail ? 1 : bsz); b++)
            if (hist_len[b] < 0 || hist_len[b] > hist_ld)
                return exl_set_err(EXL_ERR_ARG, "sample: hist_len[%d] %d outside [0, hist_ld %lld]", b, hist_len[b], (long long)hist_ld);
        for (int b = 0; b < bsz; b++) a.hist_len[b] = tail ? hist_len[0] + b : hist_len[b];
        if (tail) { a.tail = tail; a.tail_at = hist_len[0]; }
    }
    a.logits = logits; a.ld = logits_ld; a.vocab = vocab; a.slice = (vocab + SP_CL - 1) / SP_CL;
    a.hist = history; a.hist_ld = tail ? 0 : hist_ld;
    for (int b = 0; b < bsz; b++) {
        const exl_sample_params* q = per_row ? p + b : p;
        a.rp[b] = RowParams{q->temperature, q->top_k, q->top_p, q->min_p, q->typical, q->rep_penalty_max, q->rep_sustain, q->rep_decay,
                            q->bos_token_id, q->n_banned, q->banned};
    }
    a.u = u; a.tokens = tokens; a.probs = probs; a.dist = dist;

    int dev = 0;
    EXL_CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= EXL_MAX_DEVICES) return exl_set_err(EXL_ERR_ARG, "sample: device %d", dev);
    if (!g_sample_attr[dev]) {
        EXL_CUDA_TRY(cudaFuncSetAttribute(sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SP_MAX_SLICE * (int)sizeof(float)));
        g_sample_attr[dev] = true;
    }
    const size_t smem = (size_t)a.slice * sizeof(float);
    sample_kernel<<<dim3(SP_CL, bsz), SP_THREADS, smem, stream>>>(a);
    EXL_CHECK_LAUNCH("sample_kernel");
    return EXL_OK;
}

int exl_sample_launch(const float* logits, int bsz, int vocab, int64_t logits_ld, const int64_t* history, int64_t hist_ld,
                      const int* hist_len, const exl_sample_params* p, const float* u, int64_t* tokens, float* probs, float* dist,
                      cudaStream_t stream, const int64_t* tail)
{
    return sample_launch(logits, bsz, vocab, logits_ld, history, hist_ld, hist_len, p, false, u, tokens, probs, dist, stream, tail);
}

int exl_sample_rows_launch(const float* logits, int bsz, int vocab, int64_t logits_ld, const int64_t* history, int64_t hist_ld,
                           const int* hist_len, const exl_sample_params* p_rows, const float* u, int64_t* tokens, float* probs,
                           float* dist, cudaStream_t stream)
{
    return sample_launch(logits, bsz, vocab, logits_ld, history, hist_ld, hist_len, p_rows, true, u, tokens, probs, dist, stream,
                         nullptr);
}

int exl_spec_verify_launch(const float* target_logits, int k, int vocab, int64_t logits_ld, const int64_t* draft_tokens,
                           const float* draft_dist, int64_t dist_ld, const int64_t* history, int hist_len,
                           const exl_sample_params* p, const float* u, float* work, int* n_accepted, int64_t* tokens, float* probs,
                           cudaStream_t stream)
{
    if (k < 1 || k > EXL_RAGGED_MAX_SEQ - 1) return exl_set_err(EXL_ERR_ARG, "spec_verify: k %d outside [1, %d]", k, EXL_RAGGED_MAX_SEQ - 1);
    if (dist_ld < vocab) return exl_set_err(EXL_ERR_ARG, "spec_verify: dist_ld %lld < vocab %d", (long long)dist_ld, vocab);
    if (!draft_tokens || !draft_dist || !u || !work || !n_accepted || !tokens || !probs)
        return exl_set_err(EXL_ERR_ARG, "spec_verify: NULL pointer (draft_tokens %p, draft_dist %p, u %p, work %p, n_accepted %p, "
                           "tokens %p, probs %p)", (const void*)draft_tokens, (const void*)draft_dist, (const void*)u, (void*)work,
                           (void*)n_accepted, (void*)tokens, (void*)probs);
    // p_0 .. p_k: every target row through the sampler, row j's history followed by d_1 .. d_j; each row's draw with u_j lands in
    // tokens[j] / probs[j] (row k's is the bonus token), and -1 there marks an undefined row
    const int rc = exl_sample_launch(target_logits, k + 1, vocab, logits_ld, history, hist_len, history ? &hist_len : nullptr, p, u,
                                     tokens, probs, work, stream, draft_tokens);
    if (rc != EXL_OK) return rc;
    VerifyArgs a{work, draft_dist, dist_ld, draft_tokens, u, k, vocab, n_accepted, tokens, probs};
    spec_residual_kernel<<<1, SV_THREADS, 0, stream>>>(a);
    EXL_CHECK_LAUNCH("spec_residual_kernel");
    return EXL_OK;
}
