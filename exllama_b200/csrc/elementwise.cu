// elementwise.cu -- the small HBM/latency-bound ops around the q4 matmuls (stand-alone versions; the decode
// path uses the copies fused into q4_gemv.cu).  Replaces exllama_ext/cuda_func/{rms_norm.cu, rope.cu,
// column_remap.cu}, silu_mul_cuda_kernel (q4_mlp.cu:46-88) and update_cache_kernel (q4_attn.cu:19-72).
// fp16 arithmetic follows the reference instruction-for-instruction so results are bit-identical wherever the
// reference itself is deterministic.
#include "exl_common.cuh"

namespace {

// One CTA per row: fp32 sum of squares (block reduction instead of the reference's two kernels + float atomics,
// rms_norm.cu:20-79), then out = (x * half(rsqrt(sum/dim + eps))) * w with two fp16 multiplies (rms_norm.cu:113-131).
__global__ void __launch_bounds__(256) rms_norm_kernel(const half* __restrict__ x, const half* __restrict__ w,
                                                       half* __restrict__ out, float eps, float r_dim, int dim)
{
    __shared__ float s_w[8];
    __shared__ float s_tot;
    const int row = blockIdx.x, tid = threadIdx.x;
    const half* xr = x + (size_t)row * dim;
    half* orow = out + (size_t)row * dim;
    float ss = 0.f;
    const int nv = (dim % 8 == 0) ? dim / 8 : 0;     // 16-byte vector path needs every row 16-byte aligned
    for (int i = tid; i < nv; i += 256) {
        uint4 v = reinterpret_cast<const uint4*>(xr)[i];
        const half2* h = reinterpret_cast<const half2*>(&v);
        #pragma unroll
        for (int j = 0; j < 4; j++) { float2 f = __half22float2(h[j]); ss = fmaf(f.x, f.x, ss); ss = fmaf(f.y, f.y, ss); }
    }
    for (int i = nv * 8 + tid; i < dim; i += 256) { float f = __half2float(xr[i]); ss = fmaf(f, f, ss); }
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((tid & 31) == 0) s_w[tid >> 5] = ss;
    __syncthreads();
    if (tid == 0) { float t = 0.f; for (int i = 0; i < 8; i++) t += s_w[i]; s_tot = t; }
    __syncthreads();
    const half rm = __float2half_rn(rsqrtf(s_tot * r_dim + eps));
    const half2 rm2 = __half2half2(rm);
    for (int i = tid; i < nv; i += 256) {
        uint4 v = reinterpret_cast<const uint4*>(xr)[i];
        uint4 wv = reinterpret_cast<const uint4*>(w)[i];
        half2* h = reinterpret_cast<half2*>(&v);
        const half2* w2 = reinterpret_cast<const half2*>(&wv);
        #pragma unroll
        for (int j = 0; j < 4; j++) h[j] = __hmul2(__hmul2(h[j], rm2), w2[j]);
        reinterpret_cast<uint4*>(orow)[i] = v;
    }
    for (int i = nv * 8 + tid; i < dim; i += 256) orow[i] = __hmul(__hmul(xr[i], rm), w[i]);
}

// rotate-half RoPE of half2 pair c2 of one head row at position pos (rope.cu:48-67):
//   l' = hfma(l, cos_l, hmul(r, -sin_l));   r' = hfma(r, cos_r, hmul(l, sin_r))
__device__ __forceinline__ void rope_rotate(half2& l, half2& r, const half* __restrict__ sin, const half* __restrict__ cos, int pos,
                                            int c2, int head_dim)
{
    const int half_dim = head_dim / 2;
    const half2 cl = reinterpret_cast<const half2*>(cos + (size_t)pos * head_dim)[c2];
    const half2 cr = reinterpret_cast<const half2*>(cos + (size_t)pos * head_dim + half_dim)[c2];
    half2 sl = reinterpret_cast<const half2*>(sin + (size_t)pos * head_dim)[c2];
    const half2 sr = reinterpret_cast<const half2*>(sin + (size_t)pos * head_dim + half_dim)[c2];
    sl = __hneg2(sl);
    const half2 ls = __hmul2(r, sl);
    const half2 rs = __hmul2(l, sr);
    l = __hfma2(l, cl, ls);
    r = __hfma2(r, cr, rs);
}

// rotate-half RoPE in place, half2 per thread, pos = past_len + row / num_heads
__global__ void __launch_bounds__(256) rope_kernel(half* __restrict__ x, const half* __restrict__ sin, const half* __restrict__ cos,
                                                   int rows_per_batch, int head_dim, int num_heads, int past_len, long long total_pairs)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one half2 of the left half
    if (idx >= total_pairs) return;
    const int hd4 = head_dim / 4;                     // half2 per half-row
    const long long rowg = idx / hd4;                 // global row (batch * rows_per_batch + row)
    const int c2 = (int)(idx - rowg * hd4);
    const int row = (int)(rowg % rows_per_batch);
    const int pos = past_len + row / num_heads;
    half2* xl = reinterpret_cast<half2*>(x + rowg * head_dim) + c2;
    half2* xr = reinterpret_cast<half2*>(x + rowg * head_dim + head_dim / 2) + c2;
    half2 l = *xl, r = *xr;
    rope_rotate(l, r, sin, cos, pos, c2, head_dim);
    *xl = l;
    *xr = r;
}

// the sequences of a ragged batch in packed token order: sequence s owns token rows [tok0[s], tok0[s + 1])
struct RopeRagged { int n; int tok0[EXL_RAGGED_MAX_SEQ + 1]; int past[EXL_RAGGED_MAX_SEQ]; int cache[EXL_RAGGED_MAX_SEQ]; };

// One CTA per token t of sequence s, at position pos = past[s] + t - tok0[s]: rope every q head and k head of the token in place
// (rope_rotate, as rope_kernel), and write the roped k row and the v row into row pos of cache sequence cache[s].
__global__ void __launch_bounds__(256) rope_cache_ragged_kernel(half* __restrict__ q, half* __restrict__ k, const half* __restrict__ v,
                                                                half* __restrict__ kc, half* __restrict__ vc,
                                                                const half* __restrict__ sin, const half* __restrict__ cos,
                                                                const __grid_constant__ RopeRagged rr, int heads, int kv_heads, int max_seq)
{
    constexpr int HD = 128, HD4 = HD / 4;
    const int t = blockIdx.x;
    int s = 0;
    while (s + 1 < rr.n && t >= rr.tok0[s + 1]) s++;
    const int pos = rr.past[s] + t - rr.tok0[s];
    const int pairs = (heads + kv_heads) * HD4;
    for (int i = threadIdx.x; i < pairs; i += blockDim.x) {
        const int h = i / HD4, c2 = i - h * HD4;
        const bool is_k = h >= heads;
        half2* row = reinterpret_cast<half2*>(is_k ? k + ((size_t)t * kv_heads + (h - heads)) * HD : q + ((size_t)t * heads + h) * HD);
        half2 l = row[c2], r = row[HD4 + c2];
        rope_rotate(l, r, sin, cos, pos, c2, HD);
        row[c2] = l;
        row[HD4 + c2] = r;
        if (is_k) {
            const int kh = h - heads;
            const size_t dst = (((size_t)rr.cache[s] * kv_heads + kh) * max_seq + pos) * HD;
            const half2* vrow = reinterpret_cast<const half2*>(v + ((size_t)t * kv_heads + kh) * HD);
            half2* kd = reinterpret_cast<half2*>(kc + dst);
            half2* vd = reinterpret_cast<half2*>(vc + dst);
            kd[c2] = l;
            kd[HD4 + c2] = r;
            vd[c2] = vrow[c2];
            vd[HD4 + c2] = vrow[HD4 + c2];
        }
    }
}

__device__ __forceinline__ half2 silu2(half2 x)
{
    // q4_mlp.cu:38-44
    half2 one = __float2half2_rn(1.0f);
    half2 e = h2exp(__hneg2(x));
    half2 r = h2rcp(__hadd2(one, e));
    return __hmul2(x, r);
}

__global__ void __launch_bounds__(256) silu_mul_kernel(half* __restrict__ x, const half* __restrict__ y, long long n2)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n2) return;
    half2 xv = reinterpret_cast<half2*>(x)[i];
    const half2 yv = reinterpret_cast<const half2*>(y)[i];
    reinterpret_cast<half2*>(x)[i] = __hmul2(silu2(xv), yv);
}

// cache[h, past_len + t, :] = states[t, h, :]   (q4_attn.cu:32-51), 16 bytes per thread
__global__ void __launch_bounds__(256) update_cache_kernel(const half* __restrict__ ks, const half* __restrict__ vs,
                                                           half* __restrict__ kc, half* __restrict__ vc,
                                                           int head_dim, int kvh, int q_len, int max_seq, int past_len)
{
    const int hd8 = head_dim / 8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)q_len * kvh * hd8;
    if (idx >= total) return;
    const int c = (int)(idx % hd8);
    const int h = (int)((idx / hd8) % kvh);
    const int t = (int)(idx / ((long long)hd8 * kvh));
    const size_t so = ((size_t)t * kvh + h) * head_dim + (size_t)c * 8;
    const size_t co = ((size_t)h * max_seq + past_len + t) * head_dim + (size_t)c * 8;
    *reinterpret_cast<uint4*>(kc + co) = *reinterpret_cast<const uint4*>(ks + so);
    *reinterpret_cast<uint4*>(vc + co) = *reinterpret_cast<const uint4*>(vs + so);
}

// x_new[m, i] = x[m, x_map[i]]  (column_remap.cu:27-34).  One thread = one destination column, loops over a
// band of rows so x_map is read once per band.
__global__ void __launch_bounds__(256) column_remap_kernel(const half* __restrict__ x, half* __restrict__ x_new,
                                                           int M, int K, const uint32_t* __restrict__ x_map)
{
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= K) return;
    const int src = (int)x_map[col];
    const int m0 = blockIdx.y * 16, m1 = min(M, m0 + 16);
    for (int m = m0; m < m1; m++) x_new[(size_t)m * K + col] = x[(size_t)m * K + src];
}

} // namespace

int exl_rms_norm_launch(const half* x, const half* w, half* out, float eps, int rows, int dim, cudaStream_t stream)
{
    if (rows <= 0) return EXL_OK;
    rms_norm_kernel<<<rows, 256, 0, stream>>>(x, w, out, eps, 1.0f / (float)dim, dim);
    EXL_CHECK_LAUNCH("rms_norm_kernel");
    return EXL_OK;
}

int exl_rope_launch(half* x, const half* sin, const half* cos, int bsz, int rows_per_batch, int head_dim,
                    int num_heads, int past_len, cudaStream_t stream)
{
    const long long total = (long long)bsz * rows_per_batch * (head_dim / 4);
    if (total <= 0) return EXL_OK;
    if (head_dim % 4 != 0) return exl_set_err(EXL_ERR_ARG, "rope: head_dim %d must be a multiple of 4", head_dim);
    rope_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x, sin, cos, rows_per_batch, head_dim, num_heads, past_len, total);
    EXL_CHECK_LAUNCH("rope_kernel");
    return EXL_OK;
}

int exl_rope_cache_ragged_launch(half* q, half* k, const half* v, half* kc, half* vc, const half* sin, const half* cos,
                                 const exl_ragged* r, int num_cache_seqs, int heads, int kv_heads, int head_dim, int max_seq,
                                 cudaStream_t stream)
{
    const char* who = "rope_cache_ragged";
    if (!q || !k || !v || !kc || !vc || !sin || !cos)
        return exl_set_err(EXL_ERR_ARG, "%s: NULL pointer (q %p, k %p, v %p, key_cache %p, value_cache %p, sin %p, cos %p)", who,
                           (void*)q, (void*)k, (const void*)v, (void*)kc, (void*)vc, (const void*)sin, (const void*)cos);
    if (head_dim != 128) return exl_set_err(EXL_ERR_ARG, "%s: head_dim %d != 128", who, head_dim);
    if (heads < 1 || kv_heads < 1 || heads % kv_heads != 0)
        return exl_set_err(EXL_ERR_ARG, "%s: num_kv_heads %d does not divide num_heads %d", who, kv_heads, heads);
    if (const int rc = exl_ragged_validate(r, num_cache_seqs, max_seq, who)) return rc;
    RopeRagged rr;
    rr.n = r->n_seq;
    long long T = 0;
    for (int i = 0; i < r->n_seq; i++) {
        rr.tok0[i] = (int)T; rr.past[i] = r->past_len[i]; rr.cache[i] = r->cache_seq[i];
        T += r->q_len[i];
    }
    if (T > 0x7fffffffLL) return exl_set_err(EXL_ERR_ARG, "%s: %lld tokens (at most 2^31 - 1)", who, T);
    rr.tok0[r->n_seq] = (int)T;
    rope_cache_ragged_kernel<<<(unsigned)T, 256, 0, stream>>>(q, k, v, kc, vc, sin, cos, rr, heads, kv_heads, max_seq);
    EXL_CHECK_LAUNCH("rope_cache_ragged_kernel");
    return EXL_OK;
}

int exl_silu_mul_launch(half* x, const half* y, int height, int width, cudaStream_t stream)
{
    const long long n2 = (long long)height * width / 2;
    if (n2 <= 0) return EXL_OK;
    silu_mul_kernel<<<(unsigned)((n2 + 255) / 256), 256, 0, stream>>>(x, y, n2);
    EXL_CHECK_LAUNCH("silu_mul_kernel");
    return EXL_OK;
}

int exl_update_cache_launch(const half* k, const half* v, half* kc, half* vc, int head_dim, int kvh, int q_len,
                            int max_seq, int past_len, cudaStream_t stream)
{
    if (head_dim % 8 != 0) return exl_set_err(EXL_ERR_ARG, "update_cache: head_dim %d must be a multiple of 8", head_dim);
    const long long total = (long long)q_len * kvh * (head_dim / 8);
    if (total <= 0) return EXL_OK;
    update_cache_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(k, v, kc, vc, head_dim, kvh, q_len, max_seq, past_len);
    EXL_CHECK_LAUNCH("update_cache_kernel");
    return EXL_OK;
}

int exl_column_remap_launch(const half* x, half* x_new, int M, int K, const uint32_t* x_map, cudaStream_t stream)
{
    if (M <= 0) return EXL_OK;
    dim3 grid((K + 255) / 256, (M + 15) / 16);
    column_remap_kernel<<<grid, 256, 0, stream>>>(x, x_new, M, K, x_map);
    EXL_CHECK_LAUNCH("column_remap_kernel");
    return EXL_OK;
}
