/*
 * gptq_oracle.c -- CPU restatement of the exllama_ext GPTQ-4bit operator path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product path (exllama_b200/) may
 * import, link or call this file.  Allowed users: tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs.
 *
 * The reference (turboderp/exllama @ 3b013cd) ships NO CPU implementation of
 * the q4 path (exllama_ext/cpu_func holds only rep_penalty.cpp); every
 * function below restates a CUDA kernel's arithmetic on the host and cites
 * the reference file:line it follows (paths relative to the reference checkout).
 *
 * Parity pinning (every file named here exists; the GPU pins run under `pytest -m gpu` on an H100):
 *   - orc_rep_penalty / orc_apply_rep_penalty: bit-exact against the reference's own
 *     rep_penalty.cpp compiled into oracle/_ref/librep_penalty_ref.so and against
 *     tests/golden/rep_penalty_ref.npz (oracle/gen_golden_cpu.py)  -- tests/test_oracle.py.
 *   - make_x_map / make_sequential / q4_matmul (decode + reconstruct flavours): against the
 *     reference's kernels compiled for sm_90a into oracle/_ref/libexllama_ref.so, whose outputs
 *     are stored in tests/golden/ref_gpu.npz (oracle/gen_golden_ref_gpu.py)
 *     -- tests/test_gpu_q4_matmul.py::test_against_reference_*.
 *   - rms_norm, rope, column_remap, half_matmul, update_cache and silu_mul (through the fused
 *     q4_attn / q4_attn_2 / q4_mlp blocks): three-way against the same stored outputs
 *     -- tests/test_gpu_ref_pin.py.
 *   - orc_decode_attn: tests/golden/decode_attn_torch.npz (oracle/gen_golden_attn.py: the
 *     reference's attention tensor program model.py:383-409 run with torch on the CPU).
 *
 * fp16 is handled with explicit bit conversions (round-to-nearest-even) so
 * the result does not depend on the host compiler's _Float16 support.
 *
 * Build: see oracle/Makefile (gcc -O3 -march=native -fopenmp -shared -fPIC).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef uint16_t half_t;   /* IEEE binary16 bit pattern */

/* ------------------------------------------------------------------ */
/* fp16 <-> fp32/fp64 conversions                                      */
/* ------------------------------------------------------------------ */

static inline float h2f(half_t h)
{
    uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    uint32_t exp = (h >> 10) & 0x1fu;
    uint32_t man = h & 0x3ffu;
    uint32_t f;
    if (exp == 0) {
        if (man == 0) { f = sign; }
        else {
            /* subnormal: normalise */
            int e = -1;
            do { man <<= 1; e++; } while (!(man & 0x400u));
            man &= 0x3ffu;
            f = sign | ((uint32_t)(127 - 15 - e) << 23) | (man << 13);
        }
    } else if (exp == 31) {
        f = sign | 0x7f800000u | (man << 13);
    } else {
        f = sign | ((exp + 127 - 15) << 23) | (man << 13);
    }
    float out; memcpy(&out, &f, 4); return out;
}

/* double -> half, round to nearest even (single rounding from the exact double) */
static inline half_t d2h(double d)
{
    uint64_t b; memcpy(&b, &d, 8);
    uint16_t sign = (uint16_t)((b >> 48) & 0x8000u);
    int64_t exp = (int64_t)((b >> 52) & 0x7ff);
    uint64_t man = b & 0xfffffffffffffull;
    if (exp == 0x7ff) return (half_t)(sign | 0x7c00u | (man ? 0x200u : 0));
    if (exp == 0 && man == 0) return sign;
    int64_t e = exp - 1023;              /* unbiased */
    if (e > 15) return (half_t)(sign | 0x7c00u);          /* overflow -> inf */
    uint64_t m = man | (1ull << 52);     /* 53-bit significand, value = m * 2^(e-52) */
    int shift;                            /* bits to drop so that the result has 10 fraction bits */
    if (e >= -14) shift = 42;             /* normal half */
    else {
        shift = 42 + (int)(-14 - e);      /* subnormal half */
        if (shift > 63) return sign;      /* underflow to zero (far below half min subnormal / 2) */
    }
    uint64_t q = m >> shift;
    uint64_t rem = m & ((1ull << shift) - 1);
    uint64_t halfway = 1ull << (shift - 1);
    if (rem > halfway || (rem == halfway && (q & 1))) q++;
    uint16_t out;
    if (e >= -14) {
        /* q has 11 bits (1.xxxxxxxxxx) or 12 bits after carry */
        uint32_t he = (uint32_t)(e + 15);
        if (q & 0x800u) { q >>= 1; he++; }
        if (he >= 31) return (half_t)(sign | 0x7c00u);
        out = (uint16_t)((he << 10) | (q & 0x3ffu));
    } else {
        /* subnormal: q is the fraction field directly; carry into exp=1 is natural */
        out = (uint16_t)q;
    }
    return (half_t)(sign | out);
}

static inline half_t f2h(float f) { return d2h((double)f); }

/* fp16 arithmetic with one rounding, as the GPU's HMUL/HFMA/HADD do */
static inline half_t hmul(half_t a, half_t b) { return d2h((double)h2f(a) * (double)h2f(b)); }
static inline half_t hadd(half_t a, half_t b) { return d2h((double)h2f(a) + (double)h2f(b)); }
static inline half_t hfma(half_t a, half_t b, half_t c)
{
    /* product of two halves is exact in double; the sum is exact in double for
       all finite half inputs (exponent span < 53 bits) -> single rounding */
    return d2h((double)h2f(a) * (double)h2f(b) + (double)h2f(c));
}
static inline half_t hneg(half_t a) { return (half_t)(a ^ 0x8000u); }

/* exported for the python side */
float  orc_h2f(half_t h) { return h2f(h); }
half_t orc_f2h(float f)  { return f2h(f); }
half_t orc_d2h(double d) { return d2h(d); }

/* ------------------------------------------------------------------ */
/* GPTQ tensor views (exllama_ext/matrix.cuh:44-81)                    */
/*   qweight int32 [K/8, N]: nibble (k%8) of word [k/8, n]  = q[k,n]   */
/*   qzeros  int32 [G, N/8]: nibble (n%8) of word [g, n/8]  = z[g,n]   */
/*   scales  half  [G, N]                                              */
/* ------------------------------------------------------------------ */

static inline int q_at(const uint32_t* qw, int N, int k, int n)
{
    return (int)((qw[(size_t)(k >> 3) * N + n] >> ((k & 7) * 4)) & 0xf);   /* matrix.cuh:73-77 */
}
static inline int z_at(const uint32_t* qz, int N, int g, int n)
{
    return (int)((qz[(size_t)g * (N / 8) + (n >> 3)] >> ((n & 7) * 4)) & 0xf);   /* matrix.cuh:55-59 */
}

/* ------------------------------------------------------------------ */
/* act-order: x_map construction, Q4Matrix::make_sequential host part  */
/* exllama_ext/cuda_func/q4_matrix.cu:110-139                          */
/* x_map[new_row] = old_row, stable counting sort of rows by group.    */
/* (The reference routes the histogram through a `short`              */
/*  (q4_matrix.cu:122); rows-per-group <= 32767 in every real tensor,  */
/*  we reproduce the truncation for fidelity.)                         */
/* ------------------------------------------------------------------ */
void orc_make_x_map(const uint32_t* g_idx, int K, int groups, uint32_t* x_map)
{
    uint32_t* gmap = (uint32_t*)calloc((size_t)groups, sizeof(uint32_t));
    uint32_t* inv = (uint32_t*)malloc((size_t)K * sizeof(uint32_t));
    for (int i = 0; i < K; i++) gmap[g_idx[i]]++;
    uint32_t acc = 0;
    for (int i = 0; i < groups; i++) { short tmp = (short)gmap[i]; gmap[i] = acc; acc += (uint32_t)(int)tmp; }
    for (int r = 0; r < K; r++) { uint32_t g = g_idx[r]; inv[r] = gmap[g]++; }
    for (int r = 0; r < K; r++) x_map[inv[r]] = (uint32_t)r;
    free(gmap); free(inv);
}

/* make_sequential_kernel, q4_matrix.cu:61-102: new packed row r' holds the
   nibbles of original rows x_map[8r'..8r'+7]. */
void orc_make_sequential(const uint32_t* qw, uint32_t* qw_new, const uint32_t* x_map, int K, int N)
{
    #pragma omp parallel for schedule(static)
    for (int r8 = 0; r8 < K / 8; r8++) {
        for (int n = 0; n < N; n++) {
            uint32_t dst = 0;
            for (int i = 0; i < 8; i++) {
                int src_row = (int)x_map[r8 * 8 + i];
                uint32_t q = (uint32_t)q_at(qw, N, src_row, n);
                dst |= q << (i * 4);
            }
            qw_new[(size_t)r8 * N + n] = dst;
        }
    }
}

/* column_remap_kernel, column_remap.cu:7-36: x_new[m,i] = x[m, x_map[i]] */
void orc_column_remap(const half_t* x, half_t* x_new, int M, int K, const uint32_t* x_map)
{
    for (int m = 0; m < M; m++)
        for (int i = 0; i < K; i++)
            x_new[(size_t)m * K + i] = x[(size_t)m * K + x_map[i]];
}

/* ------------------------------------------------------------------ */
/* reconstruct_kernel, q4_matrix.cu:170-210:                           */
/*   out[k,n] = hmul(int2half_rn(q - (z+1)), scale[k/gs, n])           */
/* Bit-exact (one fp16 multiply of an exactly representable integer).  */
/* ------------------------------------------------------------------ */
void orc_reconstruct_f16(const uint32_t* qw, const uint32_t* qz, const half_t* scales,
                         int K, int N, int groups, half_t* out)
{
    int gs = K / groups;
    #pragma omp parallel for schedule(static)
    for (int k = 0; k < K; k++) {
        int g = k / gs;
        for (int n = 0; n < N; n++) {
            int q = q_at(qw, N, k, n) - (z_at(qz, N, g, n) + 1);
            out[(size_t)k * N + n] = hmul(d2h((double)q), scales[(size_t)g * N + n]);
        }
    }
}

/* Exact (real-valued) dequantised weight W[k,n] = scale * (q - (z+1)) in double. */
void orc_dequant_f64(const uint32_t* qw, const uint32_t* qz, const half_t* scales,
                     int K, int N, int groups, double* out)
{
    int gs = K / groups;
    #pragma omp parallel for schedule(static)
    for (int k = 0; k < K; k++) {
        int g = k / gs;
        for (int n = 0; n < N; n++) {
            int q = q_at(qw, N, k, n) - (z_at(qz, N, g, n) + 1);
            out[(size_t)k * N + n] = (double)h2f(scales[(size_t)g * N + n]) * (double)q;
        }
    }
}

/* ------------------------------------------------------------------ */
/* q4_matmul, float64 restatement ("ref64"):                           */
/*   out[m,n] (+)= sum_k x[m, map(k)] * scale[g(k),n] * (q[k,n]-(z+1)) */
/* Decode path: q4_matmul.cu:34-212 + matrix.cuh:87-133; prefill path: */
/* q4_matmul.cu:301-344.  Both compute this contraction; they differ   */
/* only in fp16 rounding/accumulation order, which is non-deterministic*/
/* in the reference (fp16 atomics).  The oracle gives the exact value. */
/* x_map may be NULL.  acc_in (may be NULL) is the pre-existing `out`  */
/* when no_zero is set (residual accumulate, q4_matmul.cu:78-82).      */
/* ------------------------------------------------------------------ */
void orc_q4_matmul_f64(const half_t* x, int M, int K, int N,
                       const uint32_t* qw, const uint32_t* qz, const half_t* scales, int groups,
                       const uint32_t* x_map, const half_t* acc_in, double* out)
{
    int gs = K / groups;
    #pragma omp parallel for schedule(static)
    for (int n = 0; n < N; n++) {
        for (int m = 0; m < M; m++) {
            double acc = 0.0;
            for (int g = 0; g < groups; g++) {
                double s = (double)h2f(scales[(size_t)g * N + n]);
                int zp = z_at(qz, N, g, n) + 1;
                double part = 0.0;
                for (int k = g * gs; k < (g + 1) * gs; k++) {
                    int kx = x_map ? (int)x_map[k] : k;
                    part += (double)h2f(x[(size_t)m * K + kx]) * (double)(q_at(qw, N, k, n) - zp);
                }
                acc += s * part;
            }
            if (acc_in) acc += (double)h2f(acc_in[(size_t)m * N + n]);
            out[(size_t)m * N + n] = acc;
        }
    }
}

/* Prefill flavour: contraction against the fp16-ROUNDED reconstructed weights
   (what cublasHgemm sees, q4_matmul.cu:323-340), accumulated exactly. */
void orc_q4_matmul_recons_f64(const half_t* x, int M, int K, int N,
                              const uint32_t* qw, const uint32_t* qz, const half_t* scales, int groups,
                              const uint32_t* x_map, const half_t* acc_in, double* out)
{
    int gs = K / groups;
    #pragma omp parallel for schedule(static)
    for (int n = 0; n < N; n++) {
        for (int m = 0; m < M; m++) {
            double acc = 0.0;
            for (int k = 0; k < K; k++) {
                int g = k / gs;
                int q = q_at(qw, N, k, n) - (z_at(qz, N, g, n) + 1);
                half_t w = hmul(d2h((double)q), scales[(size_t)g * N + n]);
                int kx = x_map ? (int)x_map[k] : k;
                acc += (double)h2f(x[(size_t)m * K + kx]) * (double)h2f(w);
            }
            if (acc_in) acc += (double)h2f(acc_in[(size_t)m * N + n]);
            out[(size_t)m * N + n] = acc;
        }
    }
}

/* ------------------------------------------------------------------ */
/* CPU baseline ("port"): dequant + fp32 GEMV, all host threads.       */
/* Restates reconstruct_kernel (q4_matrix.cu:196-208) fused with an    */
/* fp32-accumulate contraction; this is the timed cpu_baseline.        */
/* out is fp16 bits.  Row-streaming order so qweight is read once.     */
/* ------------------------------------------------------------------ */
void orc_q4_matmul_cpu_f32(const half_t* x, int M, int K, int N,
                           const uint32_t* qw, const uint32_t* qz, const half_t* scales, int groups,
                           const uint32_t* x_map, half_t* out)
{
    int gs = K / groups;
    float* xf = (float*)malloc((size_t)M * K * sizeof(float));
    for (int m = 0; m < M; m++)
        for (int k = 0; k < K; k++) {
            int kx = x_map ? (int)x_map[k] : k;
            xf[(size_t)m * K + k] = h2f(x[(size_t)m * K + kx]);
        }
    /* parallel over column blocks; each thread streams its columns over all K */
    const int NB = 64;
    #pragma omp parallel for schedule(static)
    for (int n0 = 0; n0 < N; n0 += NB) {
        int nb = (N - n0 < NB) ? (N - n0) : NB;
        float acc[8][64];
        float part[8][64];
        float sc[64]; int zp[64];
        int Mc = M < 8 ? M : 8;
        for (int m0 = 0; m0 < M; m0 += 8) {
            int mc = (M - m0 < Mc) ? (M - m0) : Mc;
            for (int m = 0; m < mc; m++) for (int j = 0; j < nb; j++) acc[m][j] = 0.f;
            for (int g = 0; g < groups; g++) {
                for (int j = 0; j < nb; j++) {
                    sc[j] = h2f(scales[(size_t)g * N + n0 + j]);
                    zp[j] = z_at(qz, N, g, n0 + j) + 1;
                }
                for (int m = 0; m < mc; m++) for (int j = 0; j < nb; j++) part[m][j] = 0.f;
                for (int k8 = g * gs / 8; k8 < (g + 1) * gs / 8; k8++) {
                    const uint32_t* wrow = qw + (size_t)k8 * N + n0;
                    for (int i = 0; i < 8; i++) {
                        int k = k8 * 8 + i;
                        for (int m = 0; m < mc; m++) {
                            float xv = xf[(size_t)(m0 + m) * K + k];
                            float* p = part[m];
                            for (int j = 0; j < nb; j++)
                                p[j] += xv * (float)((int)((wrow[j] >> (i * 4)) & 0xf) - zp[j]);
                        }
                    }
                }
                for (int m = 0; m < mc; m++) for (int j = 0; j < nb; j++) acc[m][j] += sc[j] * part[m][j];
            }
            for (int m = 0; m < mc; m++) for (int j = 0; j < nb; j++)
                out[(size_t)(m0 + m) * N + n0 + j] = f2h(acc[m][j]);
        }
    }
    free(xf);
}

/* explicit thread count (torchrun exports OMP_NUM_THREADS=1 to its children; the CPU baseline must not inherit that) */
void orc_set_num_threads(int n)
{
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int orc_num_threads(void)
{
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* ------------------------------------------------------------------ */
/* half_matmul (fp16 x fp16), exact double accumulation.               */
/* half_matmul.cu:15-54 / :119 (cublasHgemm): out (+)= x[M,K] . w[K,N] */
/* ------------------------------------------------------------------ */
void orc_half_matmul_f64(const half_t* x, const half_t* w, int M, int K, int N,
                         const half_t* acc_in, double* out)
{
    #pragma omp parallel for schedule(static)
    for (int m = 0; m < M; m++) {
        for (int n = 0; n < N; n++) {
            double acc = 0.0;
            for (int k = 0; k < K; k++)
                acc += (double)h2f(x[(size_t)m * K + k]) * (double)h2f(w[(size_t)k * N + n]);
            if (acc_in) acc += (double)h2f(acc_in[(size_t)m * N + n]);
            out[(size_t)m * N + n] = acc;
        }
    }
}

/* ------------------------------------------------------------------ */
/* rms_norm, rms_norm.cu:20-79 (row sum of squares in fp32) and        */
/* :95-152:  rm = half(rsqrtf(sum * (1/dim) + eps));                   */
/*           out = hmul(hmul(x, rm), w)                                */
/* The GPU sums in fp32 with atomics (order non-deterministic) and     */
/* uses the approximate rsqrtf; we sum in double and use 1/sqrt, so    */
/* `rm` can differ from the GPU's by 1 fp16 ulp in rare cases.         */
/* rm_out (optional) returns the per-row fp16 factor.                  */
/* ------------------------------------------------------------------ */
void orc_rms_norm(const half_t* x, const half_t* w, half_t* out, float eps, int rows, int dim, half_t* rm_out)
{
    float r_dim = 1.0f / (float)dim;
    for (int r = 0; r < rows; r++) {
        double s = 0.0;
        for (int c = 0; c < dim; c++) { double v = h2f(x[(size_t)r * dim + c]); s += v * v; }
        float sum = (float)s;
        float rmf = (float)(1.0 / sqrt((double)(sum * r_dim + eps)));
        half_t rm = f2h(rmf);
        if (rm_out) rm_out[r] = rm;
        for (int c = 0; c < dim; c++) {
            half_t m = hmul(x[(size_t)r * dim + c], rm);
            out[(size_t)r * dim + c] = hmul(m, w[c]);
        }
    }
}

/* ------------------------------------------------------------------ */
/* rope_cuda_kernel, rope.cu:20-88 (half2 path :48-67), bit-exact:     */
/*   pos = past_len + row / num_heads                                  */
/*   l' = hfma(l, cos_l, hmul(r, -sin_l));  r' = hfma(r, cos_r, hmul(l, sin_r)) */
/* x: [bsz, rows_per_batch, head_dim]; sin/cos: [max_seq, head_dim]    */
/* ------------------------------------------------------------------ */
void orc_rope(half_t* x, const half_t* sin_t, const half_t* cos_t, int bsz, int rows_per_batch,
              int head_dim, int num_heads, int past_len)
{
    int hd2 = head_dim / 2;
    for (int b = 0; b < bsz; b++)
        for (int row = 0; row < rows_per_batch; row++) {
            int pos = past_len + row / num_heads;
            half_t* xr = x + ((size_t)b * rows_per_batch + row) * head_dim;
            const half_t* sr = sin_t + (size_t)pos * head_dim;
            const half_t* cr = cos_t + (size_t)pos * head_dim;
            for (int c = 0; c < hd2; c++) {
                half_t l = xr[c], r = xr[c + hd2];
                half_t ls = hmul(r, hneg(sr[c]));
                half_t rs = hmul(l, sr[c + hd2]);
                xr[c] = hfma(l, cr[c], ls);
                xr[c + hd2] = hfma(r, cr[c + hd2], rs);
            }
        }
}

/* ------------------------------------------------------------------ */
/* silu_mul_cuda_kernel, q4_mlp.cu:27-36,46-88:                        */
/*   x = hmul(hmul(x, hrcp(hadd(1, hexp(-x)))), y)                     */
/* hexp/hrcp are approximate on the GPU (ex2.approx / rcp.approx based)*/
/* -> here each step is correctly rounded; compare with 2-ulp slack.   */
/* ------------------------------------------------------------------ */
void orc_silu_mul(half_t* x, const half_t* y, int n)
{
    half_t one = f2h(1.0f);
    for (int i = 0; i < n; i++) {
        half_t e = d2h(exp(-(double)h2f(x[i])));
        half_t s = hadd(one, e);
        half_t r = d2h(1.0 / (double)h2f(s));
        half_t v = hmul(x[i], r);
        x[i] = hmul(v, y[i]);
    }
}

/* ------------------------------------------------------------------ */
/* update_cache_kernel, q4_attn.cu:19-72:                              */
/*   cache[b, h, past_len + t, :] = states[b, t, h, :]                 */
/* states [bsz, q_len, kvh*hd]; cache [bsz_max, kvh, max_seq, hd]      */
/* (the reference kernel has no batch index: it is decode-only, bsz 1) */
/* ------------------------------------------------------------------ */
void orc_update_cache(const half_t* key, const half_t* value, half_t* kc, half_t* vc,
                      int head_dim, int kvh, int q_len, int max_seq, int past_len)
{
    for (int h = 0; h < kvh; h++)
        for (int t = 0; t < q_len; t++) {
            size_t so = (size_t)t * kvh * head_dim + (size_t)h * head_dim;
            size_t co = ((size_t)h * max_seq + past_len + t) * head_dim;
            memcpy(kc + co, key + so, (size_t)head_dim * 2);
            memcpy(vc + co, value + so, (size_t)head_dim * 2);
        }
}

/* ------------------------------------------------------------------ */
/* Decode attention, model.py:372-409 (ExLlamaAttention.fused, q_len 1, bsz 1):                    */
/*   keys/values = cache[:, :, 0:seq]; repeat_kv (model.py:327-333);                                */
/*   w = softmax(q k^T / sqrt(hd)); out[h] = w v       (out laid out [heads*hd], model.py:409)      */
/* fp16_steps == 0: everything in double (the exact answer).                                        */
/* fp16_steps == 1: the regular-attention branch's rounding points (model.py:403-406): the matmul   */
/*   result, the division and the softmax output are each rounded to fp16.                          */
/* ------------------------------------------------------------------ */
void orc_decode_attn(const half_t* q, const half_t* kc, const half_t* vc, double* out, int heads, int kv_heads,
                     int head_dim, int seq, int max_seq, int fp16_steps)
{
    const int rep = heads / kv_heads;
    double* w = (double*)malloc(sizeof(double) * (size_t)seq);
    for (int h = 0; h < heads; h++) {
        const half_t* kb = kc + (size_t)(h / rep) * max_seq * head_dim;
        const half_t* vb = vc + (size_t)(h / rep) * max_seq * head_dim;
        double mx = -1e300;
        for (int p = 0; p < seq; p++) {
            double a = 0.0;
            for (int d = 0; d < head_dim; d++) a += (double)h2f(q[(size_t)h * head_dim + d]) * (double)h2f(kb[(size_t)p * head_dim + d]);
            if (fp16_steps) { a = (double)h2f(d2h(a)); a = (double)h2f(d2h(a / (double)sqrtf((float)head_dim))); }
            else a /= sqrt((double)head_dim);
            w[p] = a;
            if (a > mx) mx = a;
        }
        double sum = 0.0;
        for (int p = 0; p < seq; p++) { w[p] = exp(w[p] - mx); sum += w[p]; }
        for (int p = 0; p < seq; p++) { w[p] /= sum; if (fp16_steps) w[p] = (double)h2f(d2h(w[p])); }
        for (int d = 0; d < head_dim; d++) {
            double a = 0.0;
            for (int p = 0; p < seq; p++) a += w[p] * (double)h2f(vb[(size_t)p * head_dim + d]);
            out[(size_t)h * head_dim + d] = a;
        }
    }
    free(w);
}

/* ------------------------------------------------------------------ */
/* rep_penalty_cpu, cpu_func/rep_penalty.cpp:5-31                      */
/* ------------------------------------------------------------------ */
void orc_rep_penalty(int vocab_size, const uint64_t* sequence, float* rep_mask,
                     float penalty_max, int sustain, int decay, int seq_len)
{
    float v = penalty_max;
    float dv = decay ? (1.0f - penalty_max) / (float)decay : 0.0f;
    int s = sustain == -1 ? seq_len : sustain;
    int beg = seq_len - s - decay;
    if (beg < 0) beg = 0;
    for (int i = 0; i < vocab_size; i++) rep_mask[i] = 1.0f;
    for (int i = seq_len; i > beg;) {
        uint64_t t = sequence[--i];
        if (v > rep_mask[t]) rep_mask[t] = v;
        if (--s < 0) v += dv;
    }
}

/* apply_rep_penalty_cpu, cpu_func/rep_penalty.cpp:36-74 (one batch row) */
void orc_apply_rep_penalty(int vocab_size, const uint64_t* sequence, float penalty_max,
                           int sustain, int decay, int seq_len, float* logits)
{
    unsigned char* seen = (unsigned char*)calloc((size_t)vocab_size, 1);
    float v = penalty_max;
    float dv = decay ? (1.0f - penalty_max) / (float)decay : 0.0f;
    int s = sustain == -1 ? seq_len : sustain;
    int beg = seq_len - s - decay;
    if (beg < 0) beg = 0;
    for (int i = seq_len; i > beg;) {
        uint64_t t = sequence[--i];
        if (!seen[t]) {
            if (logits[t] > 0.0) logits[t] /= v; else logits[t] *= v;
            seen[t] = 1;
        }
        if (--s < 0) v += dv;
    }
    free(seen);
}
