// cfg.cu -- exl_cfg_mix: classifier-free guidance (the reference's example_cfg.py:69-75) on the device, in place on the fp32 logits
// of a step: per pair (a, b), each row's repetition penalty over its own history, each row's log-softmax, and the mix
// (1 - alpha) * l_a + alpha * l_b written to both rows (include/exl_b200.h).
//
// Layout     one thread-block cluster of SP_CL CTAs per pair, with the sampler's slices (csrc/sample_select.cuh): CTA r owns the
//            slice [r * slice, (r + 1) * slice) of the vocabulary.  The two rows pass through the one slice buffer in turn: row a is
//            penalised, reduced and written back as l_a = x'_a - lse_a; row b is penalised, reduced and kept in shared memory; the
//            mix reads l_a back (L2) and writes both rows.  Shared memory stays the sampler's <= 128 KB per CTA for every vocabulary.
// Numbers    lse = m + log sum exp(x' - m) with exp and the sum in float64 (one fixed order: warp butterflies, warps in order,
//            CTAs in rank order), rounded to fp32 once; l = x' - lse, w_a * l_a and w_b * l_b and their sum each rounded to fp32
//            (no contraction).  No atomics on floating point: two calls are bitwise equal.
#include "sample_select.cuh"
#include <cmath>

namespace {

struct PairParams {
    int a, b;                    // logits rows
    float wa, wb;                // (float)(1 - alpha), (float)alpha, computed in double on the host
    float pmax; int sustain, decay;
    int len[2];                  // history lengths of rows a and b (0: no penalty)
};

struct CfgArgs {
    float* logits; int64_t ld; int vocab; int slice;
    const int64_t* hist; int64_t hist_ld;
    PairParams pr[EXL_CFG_MAX_PAIRS];            // a cluster is one pair, so every branch on a pair's values is uniform in it
};
static_assert(sizeof(CfgArgs) <= 4096, "CfgArgs must fit the classic 4 KB kernel parameter space");

__global__ void __cluster_dims__(SP_CL, 1, 1) __launch_bounds__(SP_THREADS, 1) cfg_mix_kernel(const __grid_constant__ CfgArgs a)
{
    extern __shared__ __align__(16) float s_row[];
    __shared__ Shared sh;
    int* s_int = reinterpret_cast<int*>(s_row);
    cg::cluster_group cluster = cg::this_cluster();
    const PairParams& pp = a.pr[blockIdx.y];
    const int rank = (int)cluster.block_rank();
    const int lo = rank * a.slice;
    const int n = max(0, min(a.slice, a.vocab - lo));
    const float dv = pp.decay ? (1.0f - pp.pmax) / (float)pp.decay : 0.0f;
    float* la = a.logits + (int64_t)pp.a * a.ld + lo;
    float* lb = a.logits + (int64_t)pp.b * a.ld + lo;
    int ph = 0;
    int undefined = 0;
    float lse_a = 0.0f, lse_b = 0.0f;
    for (int side = 0; side < 2; side++) {
        const int row = side ? pp.b : pp.a;
        float* lg = side ? lb : la;
        int bad = 0;
        __syncthreads();                                             // the slice buffer is free again
        // 1. penalised logits x' of the slice into shared memory
        const bool pen = a.hist != nullptr && pp.pmax != 1.0f && pp.len[side] > 0;
        long long s0 = 0;
        if (pen)
            s0 = penalty_scan(sh, s_int, a.hist + (int64_t)row * a.hist_ld, nullptr, 0, pp.len[side], pp.pmax, pp.sustain, pp.decay, dv,
                              a.vocab, lo, n, bad);
        float mx = -INFINITY;
        for (int i = threadIdx.x; i < n; i += SP_THREADS) {
            float x = lg[i];
            if (pen) x = penalise(sh, x, s_int[i], s0, dv);
            s_row[i] = x;
            if (isnan(x)) bad = 1;
            mx = fmaxf(mx, x);
        }
        // 2. the row maximum and the undefined test, over the cluster
        {
            Part p{}; p.f = block_max_f(mx, sh); p.bad = block_or(bad, sh);
            cluster_exchange(sh, ph, p, [](const Part* ps, Part& o) {
                float m = -INFINITY; int b = 0;
                for (int r = 0; r < SP_CL; r++) { m = fmaxf(m, ps[r].f); b |= ps[r].bad; }
                o.f = m; o.bad = b;
            });
            mx = sh.bc.f; bad = sh.bc.bad;
        }
        if (bad || mx == -INFINITY) { undefined = 1; break; }        // the same decision in every CTA of the cluster
        // 3. lse = m + log sum exp(x' - m), float64, rounded to fp32 once
        double z = 0.0;
        for (int i = threadIdx.x; i < n; i += SP_THREADS) z += exp((double)s_row[i] - (double)mx);
        z = cluster_sum_d(sh, ph, z);
        (side ? lse_b : lse_a) = (float)((double)mx + log(z));
        // row a: l_a goes back to the logits; it is read again, by the thread that wrote it, in the mix
        if (side == 0)
            for (int i = threadIdx.x; i < n; i += SP_THREADS) la[i] = __fsub_rn(s_row[i], lse_a);
    }
    if (undefined) {
        for (int i = threadIdx.x; i < n; i += SP_THREADS) { la[i] = NAN; lb[i] = NAN; }
    } else {
        // 4. the mix, written to both rows
        for (int i = threadIdx.x; i < n; i += SP_THREADS) {
            const float lbi = __fsub_rn(s_row[i], lse_b);
            const float m = __fadd_rn(__fmul_rn(pp.wa, la[i]), __fmul_rn(pp.wb, lbi));
            la[i] = m;
            lb[i] = m;
        }
    }
    cluster.sync();                                                  // no CTA leaves while another may read its exchange slot
}

bool g_cfg_attr[EXL_MAX_DEVICES];

} // namespace

int exl_cfg_mix_launch(float* logits, int rows, int vocab, int64_t ld, const int64_t* history, int64_t hist_ld, const int* hist_len,
                       const exl_cfg_pair* pairs, int n_pairs, cudaStream_t stream)
{
    if (!logits || !pairs)
        return exl_set_err(EXL_ERR_ARG, "cfg_mix: NULL pointer (logits %p, pairs_host %p)", (void*)logits, (const void*)pairs);
    if (rows < 1 || rows > EXL_RAGGED_MAX_SEQ) return exl_set_err(EXL_ERR_ARG, "cfg_mix: rows %d outside [1, %d]", rows, EXL_RAGGED_MAX_SEQ);
    if (vocab < 1 || vocab > SP_MAX_VOCAB) return exl_set_err(EXL_ERR_ARG, "cfg_mix: vocab %d outside [1, %d]", vocab, SP_MAX_VOCAB);
    if (ld < vocab) return exl_set_err(EXL_ERR_ARG, "cfg_mix: ld %lld < vocab %d", (long long)ld, vocab);
    if (n_pairs < 1 || n_pairs > EXL_CFG_MAX_PAIRS)
        return exl_set_err(EXL_ERR_ARG, "cfg_mix: n_pairs %d outside [1, %d]", n_pairs, EXL_CFG_MAX_PAIRS);
    if (history) {
        if (!hist_len) return exl_set_err(EXL_ERR_ARG, "cfg_mix: history without hist_len_host");
        for (int r = 0; r < rows; r++)
            if (hist_len[r] < 0 || hist_len[r] > hist_ld)
                return exl_set_err(EXL_ERR_ARG, "cfg_mix: hist_len[%d] %d outside [0, hist_ld %lld]", r, hist_len[r], (long long)hist_ld);
    }
    CfgArgs args{};
    int owner[EXL_RAGGED_MAX_SEQ];
    for (int r = 0; r < rows; r++) owner[r] = -1;
    for (int k = 0; k < n_pairs; k++) {
        const exl_cfg_pair& q = pairs[k];
        for (int side = 0; side < 2; side++) {
            const int r = side ? q.b : q.a;
            if (r < 0 || r >= rows) return exl_set_err(EXL_ERR_ARG, "cfg_mix: pair %d: row %s %d outside [0, rows %d)", k, side ? "b" : "a", r, rows);
        }
        if (q.a == q.b) return exl_set_err(EXL_ERR_ARG, "cfg_mix: pair %d: a == b == %d", k, q.a);
        for (int side = 0; side < 2; side++) {
            const int r = side ? q.b : q.a;
            if (owner[r] >= 0) return exl_set_err(EXL_ERR_ARG, "cfg_mix: pair %d: row %d is already in pair %d", k, r, owner[r]);
            owner[r] = k;
        }
        if (!std::isfinite(q.alpha)) return exl_set_err(EXL_ERR_ARG, "cfg_mix: pair %d: alpha %g is not finite", k, q.alpha);
        if (q.rep_sustain < -1) return exl_set_err(EXL_ERR_ARG, "cfg_mix: pair %d: rep_sustain %d < -1", k, q.rep_sustain);
        if (q.rep_decay < 0) return exl_set_err(EXL_ERR_ARG, "cfg_mix: pair %d: rep_decay %d < 0", k, q.rep_decay);
        PairParams& p = args.pr[k];
        p.a = q.a; p.b = q.b;
        p.wa = (float)(1.0 - q.alpha); p.wb = (float)q.alpha;
        p.pmax = q.rep_penalty_max; p.sustain = q.rep_sustain; p.decay = q.rep_decay;
        p.len[0] = history ? hist_len[q.a] : 0;
        p.len[1] = history ? hist_len[q.b] : 0;
    }
    args.logits = logits; args.ld = ld; args.vocab = vocab; args.slice = (vocab + SP_CL - 1) / SP_CL;
    args.hist = history; args.hist_ld = hist_ld;

    int dev = 0;
    EXL_CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= EXL_MAX_DEVICES) return exl_set_err(EXL_ERR_ARG, "cfg_mix: device %d", dev);
    if (!g_cfg_attr[dev]) {
        EXL_CUDA_TRY(cudaFuncSetAttribute(cfg_mix_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SP_MAX_SLICE * (int)sizeof(float)));
        g_cfg_attr[dev] = true;
    }
    cfg_mix_kernel<<<dim3(SP_CL, n_pairs), SP_THREADS, (size_t)args.slice * sizeof(float), stream>>>(args);
    EXL_CHECK_LAUNCH("cfg_mix_kernel");
    return EXL_OK;
}
