// prefill_attn.cu -- causal attention of a prompt chunk over the KV cache, read in place (prefill at any past_len).
//
// Replaces repeat_kv + the additive causal mask + scaled_dot_product_attention of ExLlamaAttention.forward (model.py:447-493,
// mask model.py:1016-1018) for a chunk of q_len tokens at positions [past_len, past_len + q_len):
//
//   out[b, t, h, :] = softmax_j(q[b, t, h] . K[b, kvh(h), j] / sqrt(128)) . V[b, kvh(h), j],   j in [0, past_len + t]
//
// FlashAttention-2 schedule on mma.sync.m16n8k16 (f16 in, f32 accumulate):
//   rows     a query tile is 64 ROWS of one KV group, row r = (token r / n_rep, query head r % n_rep of the group): under
//            grouped-query attention the n_rep heads that share a KV head share every K/V tile, which is loaded once per group
//            and not once per head, and no repeat_kv copy exists
//   CTA      4 warps x 16 rows; each CTA takes its (sequence, KV group, row tile) from the launch's work description
//            (prefill_attn_sched.h): grid (kv_heads * bsz, row tiles) for a uniform batch (exl_prefill_attn), one CTA per tile of
//            every sequence for a ragged batch (exl_prefill_attn_ragged, no CTA for padding, the sequences with the most keys
//            first); row tiles in reverse so the longest rows start first; the math inside a tile is the same for both
//   K / V    64-key tiles, double-buffered through cp.async (zero-filled past the CTA's last visible key: a cache row that was
//            never written, NaN included, is never read); ldmatrix from XOR-swizzled shared memory (conflict-free phases)
//   softmax  online, fp32 scores / max / sum / output accumulators; P rounded to fp16 for the P . V product; only the key
//            tiles that cross the diagonal are masked, tiles entirely above it are never loaded
//   output   one fp16 rounding of o / l, written straight into [tokens, heads * 128] (o_proj's input layout)
// No atomics and a fixed reduction order: two launches are bitwise equal.  No programmatic dependent launch.
#include "exl_common.cuh"
#include "prefill_attn_sched.h"

static_assert(pa_sched::MAX_SEQ == EXL_RAGGED_MAX_SEQ, "one ragged description holds every sequence exl_ragged may name");

namespace {

constexpr int PA_THREADS = 128;                          // 4 warps x 16 query rows
constexpr int PA_BM = pa_sched::BM;                      // query rows per CTA
constexpr int PA_BN = 64;                                // keys per K / V tile
constexpr int HD = 128;
constexpr uint32_t PA_TILE_BYTES = 64 * HD * 2;          // one [64][128] fp16 tile
constexpr size_t PA_SMEM = 5 * (size_t)PA_TILE_BYTES;    // Q, K[2], V[2] = 80 KB (two CTAs per SM)

__device__ __forceinline__ uint32_t pa_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// byte offset of 16-byte chunk c (0..15) of row r of a [64][128] half tile; the chunk index is XORed with r & 7 so the eight rows
// one ldmatrix phase reads land in eight different bank groups
__device__ __forceinline__ uint32_t pa_off(int r, int c) { return (uint32_t)(r * HD + ((c ^ (r & 7)) << 3)) * 2u; }

// 16 bytes global -> shared, or 16 zero bytes without reading global memory (src-size 0)
__device__ __forceinline__ void pa_cp16(uint32_t dst, const half* src, bool valid)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" :: "r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}

__device__ __forceinline__ void pa_ldsm4(uint32_t* r, uint32_t addr)
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}

__device__ __forceinline__ void pa_ldsm4_t(uint32_t* r, uint32_t addr)
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}

__device__ __forceinline__ void pa_mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t pa_pack(float lo, float hi)
{
    const half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}

__global__ void __launch_bounds__(PA_THREADS, 2) prefill_attn_kernel(const half* __restrict__ q, const half* __restrict__ kc,
                                                                  const half* __restrict__ vc, half* __restrict__ out,
                                                                  const __grid_constant__ pa_sched::Work work, int heads,
                                                                  int max_seq, float scale_log2)
{
    extern __shared__ __align__(128) unsigned char pa_sm[];
    const uint32_t sQ = pa_smem(pa_sm);
    const uint32_t sK = sQ + PA_TILE_BYTES;              // K[0], K[1]
    const uint32_t sV = sQ + 3 * PA_TILE_BYTES;          // V[0], V[1]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int kv_heads = work.kv_heads, n_rep = work.n_rep;
    const pa_sched::Tile tile = pa_sched::tile_of(work, (int)blockIdx.x, (int)blockIdx.y);
    const int g = tile.g, past_len = tile.past_len, m0 = tile.m0;
    const int R = tile.q_len * n_rep;                     // rows of this (sequence, KV group)
    const int t_lo = m0 / n_rep, t_hi = (min(R, m0 + PA_BM) - 1) / n_rep;
    const int kv_end = past_len + t_hi + 1;               // keys any row of this CTA sees
    const int n_tiles = (kv_end + PA_BN - 1) / PA_BN;
    const int diag = past_len + t_lo;                     // a key tile ending at or before this key needs no mask
    const size_t cache_off = ((size_t)tile.cache_seq * kv_heads + g) * max_seq * HD;
    const half* kbase = kc + cache_off;
    const half* vbase = vc + cache_off;
    const size_t qrow0 = (size_t)tile.tok0 * heads + (size_t)g * n_rep;   // (token 0, first head of the group) of this sequence

    // ---- Q tile (rows past R zero-filled) and K / V tile 0 ----
    #pragma unroll
    for (int i = 0; i < 8; i++) {
        const int idx = tid + i * PA_THREADS, r = idx >> 4, c = idx & 15;
        const int gr = m0 + r;
        const bool valid = gr < R;
        const half* src = q;
        if (valid) {
            const int t = gr / n_rep;
            src = q + (qrow0 + (size_t)t * heads + (gr - t * n_rep)) * HD + c * 8;
        }
        pa_cp16(sQ + pa_off(r, c), src, valid);
    }
    auto load_kv = [&](int tile, int buf) {
        #pragma unroll
        for (int i = 0; i < 8; i++) {
            const int idx = tid + i * PA_THREADS, r = idx >> 4, c = idx & 15;
            const int j = tile * PA_BN + r;
            const bool valid = j < kv_end;
            const size_t off = valid ? (size_t)j * HD + c * 8 : 0;
            pa_cp16(sK + buf * PA_TILE_BYTES + pa_off(r, c), kbase + off, valid);
            pa_cp16(sV + buf * PA_TILE_BYTES + pa_off(r, c), vbase + off, valid);
        }
    };
    load_kv(0, 0);
    asm volatile("cp.async.commit_group;" ::: "memory");

    // this thread's two rows (lane / 4 and lane / 4 + 8 of the warp's 16) and the last key each may see
    const int rowA = m0 + warp * 16 + (lane >> 2), rowB = rowA + 8;
    const int limA = past_len + min(rowA, R - 1) / n_rep;
    const int limB = past_len + min(rowB, R - 1) / n_rep;

    uint32_t qf[8][4];                                    // A fragments of the warp's 16 x 128 Q slice
    float o[16][4];
    #pragma unroll
    for (int d = 0; d < 16; d++) o[d][0] = o[d][1] = o[d][2] = o[d][3] = 0.f;
    float mA = -INFINITY, mB = -INFINITY, lA = 0.f, lB = 0.f;   // running max (raw score units) and per-thread partial sums

    for (int n = 0; n < n_tiles; n++) {
        if (n + 1 < n_tiles) load_kv(n + 1, (n + 1) & 1);
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        __syncthreads();
        if (n == 0) {
            #pragma unroll
            for (int kk = 0; kk < 8; kk++) pa_ldsm4(qf[kk], sQ + pa_off(warp * 16 + (lane & 15), kk * 2 + (lane >> 4)));
        }
        const uint32_t kb = sK + (n & 1) * PA_TILE_BYTES, vb = sV + (n & 1) * PA_TILE_BYTES;

        // ---- S = Q K^T: 16 rows x 64 keys per warp ----
        float s[8][4];
        #pragma unroll
        for (int j = 0; j < 8; j++) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
        #pragma unroll
        for (int kk = 0; kk < 8; kk++) {
            #pragma unroll
            for (int np = 0; np < 4; np++) {
                uint32_t bf[4];
                pa_ldsm4(bf, kb + pa_off(np * 16 + (lane & 7) + ((lane >> 4) << 3), kk * 2 + ((lane >> 3) & 1)));
                pa_mma(s[2 * np], qf[kk], bf[0], bf[1]);
                pa_mma(s[2 * np + 1], qf[kk], bf[2], bf[3]);
            }
        }

        // ---- causal mask (diagonal tiles only) and online softmax ----
        const int kstart = n * PA_BN;
        if (kstart + PA_BN - 1 > diag) {
            #pragma unroll
            for (int j = 0; j < 8; j++) {
                #pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int key = kstart + j * 8 + (lane & 3) * 2 + e;
                    if (key > limA) s[j][e] = -INFINITY;
                    if (key > limB) s[j][2 + e] = -INFINITY;
                }
            }
        }
        float xA = mA, xB = mB;
        #pragma unroll
        for (int j = 0; j < 8; j++) {
            xA = fmaxf(xA, fmaxf(s[j][0], s[j][1]));
            xB = fmaxf(xB, fmaxf(s[j][2], s[j][3]));
        }
        xA = fmaxf(xA, __shfl_xor_sync(0xffffffffu, xA, 1)); xA = fmaxf(xA, __shfl_xor_sync(0xffffffffu, xA, 2));
        xB = fmaxf(xB, __shfl_xor_sync(0xffffffffu, xB, 1)); xB = fmaxf(xB, __shfl_xor_sync(0xffffffffu, xB, 2));
        // key 0 is visible to every row and sits in tile 0, so the max is finite from the first tile on
        const float alphaA = exp2f((mA - xA) * scale_log2), alphaB = exp2f((mB - xB) * scale_log2);   // 0 on tile 0
        mA = xA; mB = xB;
        const float sA = xA * scale_log2, sB = xB * scale_log2;
        lA *= alphaA; lB *= alphaB;
        #pragma unroll
        for (int d = 0; d < 16; d++) { o[d][0] *= alphaA; o[d][1] *= alphaA; o[d][2] *= alphaB; o[d][3] *= alphaB; }
        uint32_t pf[4][4];                                // A fragments of P (fp16), one per 16 keys
        #pragma unroll
        for (int j = 0; j < 8; j++) {
            const float p0 = exp2f(fmaf(s[j][0], scale_log2, -sA)), p1 = exp2f(fmaf(s[j][1], scale_log2, -sA));
            const float p2 = exp2f(fmaf(s[j][2], scale_log2, -sB)), p3 = exp2f(fmaf(s[j][3], scale_log2, -sB));
            lA += p0 + p1; lB += p2 + p3;
            pf[j >> 1][(j & 1) * 2] = pa_pack(p0, p1);
            pf[j >> 1][(j & 1) * 2 + 1] = pa_pack(p2, p3);
        }

        // ---- O += P V ----
        #pragma unroll
        for (int kk = 0; kk < 4; kk++) {
            #pragma unroll
            for (int dp = 0; dp < 8; dp++) {
                uint32_t bf[4];
                pa_ldsm4_t(bf, vb + pa_off(kk * 16 + (lane & 7) + (((lane >> 3) & 1) << 3), dp * 2 + (lane >> 4)));
                pa_mma(o[2 * dp], pf[kk], bf[0], bf[1]);
                pa_mma(o[2 * dp + 1], pf[kk], bf[2], bf[3]);
            }
        }
        __syncthreads();                                  // buffer n & 1 is refilled by the next iteration's load
    }

    lA += __shfl_xor_sync(0xffffffffu, lA, 1); lA += __shfl_xor_sync(0xffffffffu, lA, 2);
    lB += __shfl_xor_sync(0xffffffffu, lB, 1); lB += __shfl_xor_sync(0xffffffffu, lB, 2);
    const float iA = 1.f / lA, iB = 1.f / lB;
    const int col = (lane & 3) * 2;
    if (rowA < R) {
        const int t = rowA / n_rep;
        half* dst = out + (qrow0 + (size_t)t * heads + (rowA - t * n_rep)) * HD + col;
        #pragma unroll
        for (int d = 0; d < 16; d++) *reinterpret_cast<half2*>(dst + d * 8) = __floats2half2_rn(o[d][0] * iA, o[d][1] * iA);
    }
    if (rowB < R) {
        const int t = rowB / n_rep;
        half* dst = out + (qrow0 + (size_t)t * heads + (rowB - t * n_rep)) * HD + col;
        #pragma unroll
        for (int d = 0; d < 16; d++) *reinterpret_cast<half2*>(dst + d * 8) = __floats2half2_rn(o[d][2] * iB, o[d][3] * iB);
    }
}

} // namespace

// one launch of prefill_attn_kernel over a validated work description
static int pa_launch(const half* q, const half* kc, const half* vc, half* out, const pa_sched::Work& work, int heads, int max_seq,
                     cudaStream_t stream)
{
    int dev = 0;
    EXL_CUDA_TRY(cudaGetDevice(&dev));
    static bool attr_done[EXL_MAX_DEVICES] = {};
    if (dev >= 0 && dev < EXL_MAX_DEVICES && !attr_done[dev]) {
        EXL_CUDA_TRY(cudaFuncSetAttribute(prefill_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PA_SMEM));
        attr_done[dev] = true;
    }
    const float scale_log2 = 1.4426950408889634f / sqrtf((float)HD);
    const dim3 grid((unsigned)pa_sched::grid_x(work), (unsigned)pa_sched::grid_y(work));
    prefill_attn_kernel<<<grid, PA_THREADS, PA_SMEM, stream>>>(q, kc, vc, out, work, heads, max_seq, scale_log2);
    EXL_CHECK_LAUNCH("prefill_attn_kernel");
    return EXL_OK;
}

int exl_prefill_attn_launch(const half* q, const half* kc, const half* vc, half* out, int bsz, int q_len, int heads, int kv_heads,
                            int head_dim, int past_len, int max_seq, cudaStream_t stream)
{
    if (!q || !kc || !vc || !out)
        return exl_set_err(EXL_ERR_ARG, "prefill_attn: NULL pointer (q %p, key_cache %p, value_cache %p, out %p)",
                           (const void*)q, (const void*)kc, (const void*)vc, (void*)out);
    if (head_dim != HD) return exl_set_err(EXL_ERR_ARG, "prefill_attn: head_dim %d != 128", head_dim);
    if (heads < 1 || kv_heads < 1 || heads % kv_heads != 0)
        return exl_set_err(EXL_ERR_ARG, "prefill_attn: num_kv_heads %d does not divide num_heads %d", kv_heads, heads);
    if (bsz < 1) return exl_set_err(EXL_ERR_ARG, "prefill_attn: bsz %d < 1", bsz);
    if (q_len < 1) return exl_set_err(EXL_ERR_ARG, "prefill_attn: q_len %d < 1", q_len);
    if (past_len < 0) return exl_set_err(EXL_ERR_ARG, "prefill_attn: past_len %d < 0", past_len);
    if (max_seq < 1 || (long long)past_len + q_len > max_seq)
        return exl_set_err(EXL_ERR_ARG, "prefill_attn: past_len %d + q_len %d > max_seq_len %d", past_len, q_len, max_seq);
    const long long rows = (long long)q_len * (heads / kv_heads);
    const long long row_tiles = (rows + PA_BM - 1) / PA_BM;
    if (row_tiles > 65535 || (long long)bsz * kv_heads > 0x7fffffffLL)
        return exl_set_err(EXL_ERR_ARG, "prefill_attn: q_len %d x %d heads per KV head needs %lld row tiles (at most 65535)",
                           q_len, heads / kv_heads, row_tiles);
    pa_sched::Work work;
    pa_sched::make_uniform(work, bsz, q_len, past_len, kv_heads, heads / kv_heads);
    return pa_launch(q, kc, vc, out, work, heads, max_seq, stream);
}

int exl_ragged_validate(const exl_ragged* r, int num_cache_seqs, int max_seq, const char* who)
{
    if (!r || !r->q_len || !r->past_len || !r->cache_seq)
        return exl_set_err(EXL_ERR_ARG, "%s: NULL pointer (ragged %p, q_len %p, past_len %p, cache_seq %p)", who, (const void*)r,
                           r ? (const void*)r->q_len : nullptr, r ? (const void*)r->past_len : nullptr,
                           r ? (const void*)r->cache_seq : nullptr);
    if (r->n_seq < 1 || r->n_seq > EXL_RAGGED_MAX_SEQ)
        return exl_set_err(EXL_ERR_ARG, "%s: n_seq %d outside [1, %d]", who, r->n_seq, EXL_RAGGED_MAX_SEQ);
    for (int i = 0; i < r->n_seq; i++) {
        const int ql = r->q_len[i], pl = r->past_len[i], cs = r->cache_seq[i];
        if (ql < 1) return exl_set_err(EXL_ERR_ARG, "%s: q_len[%d] %d < 1", who, i, ql);
        if (pl < 0) return exl_set_err(EXL_ERR_ARG, "%s: past_len[%d] %d < 0", who, i, pl);
        if ((long long)pl + ql > max_seq)
            return exl_set_err(EXL_ERR_ARG, "%s: past_len[%d] %d + q_len[%d] %d > max_seq_len %d", who, i, pl, i, ql, max_seq);
        if (cs < 0 || cs >= num_cache_seqs)
            return exl_set_err(EXL_ERR_ARG, "%s: cache_seq[%d] %d outside [0, num_cache_seqs %d)", who, i, cs, num_cache_seqs);
        for (int j = 0; j < i; j++)
            if (r->cache_seq[j] == cs) return exl_set_err(EXL_ERR_ARG, "%s: cache_seq[%d] %d repeats cache_seq[%d]", who, i, cs, j);
    }
    return EXL_OK;
}

int exl_prefill_attn_ragged_launch(const half* q, const half* kc, const half* vc, half* out, const exl_ragged* r, int num_cache_seqs,
                                   int heads, int kv_heads, int head_dim, int max_seq, cudaStream_t stream)
{
    const char* who = "prefill_attn_ragged";
    if (!q || !kc || !vc || !out)
        return exl_set_err(EXL_ERR_ARG, "%s: NULL pointer (q %p, key_cache %p, value_cache %p, out %p)", who,
                           (const void*)q, (const void*)kc, (const void*)vc, (void*)out);
    if (head_dim != HD) return exl_set_err(EXL_ERR_ARG, "%s: head_dim %d != 128", who, head_dim);
    if (heads < 1 || kv_heads < 1 || heads % kv_heads != 0)
        return exl_set_err(EXL_ERR_ARG, "%s: num_kv_heads %d does not divide num_heads %d", who, kv_heads, heads);
    if (const int rc = exl_ragged_validate(r, num_cache_seqs, max_seq, who)) return rc;
    long long ctas = 0;
    for (int i = 0; i < r->n_seq; i++) ctas += (long long)kv_heads * pa_sched::row_tiles_of(r->q_len[i], heads / kv_heads);
    if (ctas > 0x7fffffffLL) return exl_set_err(EXL_ERR_ARG, "%s: %lld CTAs (at most 2^31 - 1)", who, ctas);
    pa_sched::Work work;
    pa_sched::make_ragged(work, r->n_seq, r->q_len, r->past_len, r->cache_seq, kv_heads, heads / kv_heads);
    return pa_launch(q, kc, vc, out, work, heads, max_seq, stream);
}
