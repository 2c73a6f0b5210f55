// extern "C" shim over the reference's OWN CUDA kernels (exllama_ext/cuda_func/*.cu,
// cuda_buffers.cu), compiled unmodified from the reference checkout for sm_90a into
// oracle/_ref/libexllama_ref.so (see oracle/Makefile).  This is the live GPU
// oracle (oracle/gen_golden_ref_gpu.py).  TEST INFRASTRUCTURE ONLY -- never loaded by the product.
//
// The entry points mirror include/exl_b200.h so tests can drive both libraries
// with the same arguments.  All reference kernels run on the legacy default stream.
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cublas_v2.h>
#include <cstdint>
#include "tuning.h"
#include "cuda_buffers.cuh"
#include "cuda_func/q4_matrix.cuh"
#include "cuda_func/q4_matmul.cuh"
#include "cuda_func/column_remap.cuh"
#include "cuda_func/rms_norm.cuh"
#include "cuda_func/rope.cuh"
#include "cuda_func/half_matmul.cuh"
#include "cuda_func/q4_attn.cuh"
#include "cuda_func/q4_mlp.cuh"

static ExLlamaTuning g_tuning = {8, 2, 8, false, false, false, false, false, false};
static cublasHandle_t g_handle = nullptr;
static cublasHandle_t handle() { if (!g_handle) cublasCreate(&g_handle); return g_handle; }

extern "C" {

void ref_set_tuning_params(int recons_thd, int fused_mlp_thd, int sdp_thd, int fused_remap,
                           int rms_nh2, int rope_nh2, int mm_nh2, int silu_nh2, int conc)
{
    g_tuning.matmul_recons_thd = recons_thd; g_tuning.fused_mlp_thd = fused_mlp_thd; g_tuning.sdp_thd = sdp_thd;
    g_tuning.matmul_fused_remap = fused_remap; g_tuning.rmsnorm_no_half2 = rms_nh2; g_tuning.rope_no_half2 = rope_nh2;
    g_tuning.matmul_no_half2 = mm_nh2; g_tuning.silu_no_half2 = silu_nh2; g_tuning.concurrent_streams = conc;
}

void ref_prepare_buffers(int device, void* temp_state, int temp_state_numel, void* temp_mlp,
                         void* temp_zeros_float, void* temp_dq, int max_zeros_float)
{
    prepare_buffers_cuda(device, (half*)temp_state, temp_state_numel, (half*)temp_mlp,
                         (float*)temp_zeros_float, (half*)temp_dq, max_zeros_float);
}

void ref_cleanup() { cleanup_buffers_cuda(); g_q4_free_matrices(); }

// g_idx_host: int32 [K] on the HOST or NULL.  Overwrites qweight in place when given (as the reference does).
void* ref_make_q4(void* qweight, void* qzeros, void* scales, const void* g_idx_host,
                  int K, int N, int groups, int device)
{
    Q4Matrix* m = new Q4Matrix(K, N, groups, (uint32_t*)qweight, (uint32_t*)qzeros, (half*)scales,
                               (uint32_t*)g_idx_host, device);
    g_q4_keep_matrix(m);
    return (void*)m;
}

int ref_q4_has_x_map(void* w) { return ((Q4Matrix*)w)->cuda_x_map != nullptr; }
void ref_q4_get_x_map(void* w, void* out_host)
{
    Q4Matrix* m = (Q4Matrix*)w;
    cudaMemcpy(out_host, m->cuda_x_map, (size_t)m->height * 4, cudaMemcpyDeviceToHost);
}

// mode 0: decode kernel (q4_matmul_cuda); mode 1: reconstruct + cublasHgemm (q4_matmul_recons_cuda)
void ref_q4_matmul(const void* x, int M, void* w, void* out, int no_zero, int mode)
{
    if (mode == 0) q4_matmul_cuda(&g_tuning, (const half*)x, M, (Q4Matrix*)w, (half*)out, no_zero != 0);
    else           q4_matmul_recons_cuda(&g_tuning, (const half*)x, M, (Q4Matrix*)w, (half*)out, handle(), no_zero != 0);
}

void ref_reconstruct(void* w, void* out) { ((Q4Matrix*)w)->reconstruct((half*)out); }

void ref_column_remap(const void* x, void* x_new, int M, int K, const void* x_map)
{ column_remap_cuda((const half*)x, (half*)x_new, M, K, (const uint32_t*)x_map); }

void ref_rms_norm(void* x, const void* w, void* out, float eps, int rows, int dim, int device)
{ rms_norm_cuda(&g_tuning, (half*)x, (const half*)w, (half*)out, eps, rows, dim, device); }

void ref_rope(void* x, const void* sin, const void* cos, int bsz, int rows_per_batch, int head_dim,
              int num_heads, int past_len)
{ rope_cuda(&g_tuning, (half*)x, (const half*)sin, (const half*)cos, bsz, rows_per_batch, head_dim, num_heads, past_len); }

void ref_half_matmul(const void* x, const void* w, void* out, int M, int K, int N)
{ half_matmul_cuda((const half*)x, (const half*)w, (half*)out, M, K, N); }

void ref_half_matmul_cublas(const void* x, const void* w, void* out, int M, int K, int N, int no_zero)
{ half_matmul_cublas_cuda(&g_tuning, (const half*)x, (const half*)w, (half*)out, M, K, N, handle(), no_zero != 0); }

void ref_q4_attn(void* x, const void* rms_w, float eps, void* q, void* k, void* v,
                 void* q_proj, void* k_proj, void* v_proj, void* sin, void* cos,
                 int bsz, int q_len, int dim, int head_dim, int num_heads, int num_kv_heads, int past_len,
                 void* key_cache, void* value_cache, int max_seq_len, int device)
{
    q4_attn_cuda(&g_tuning, 0, handle(), (half*)x, (const half*)rms_w, eps, (half*)q, (half*)k, (half*)v,
                 (Q4Matrix*)q_proj, (Q4Matrix*)k_proj, (Q4Matrix*)v_proj, (half*)sin, (half*)cos,
                 bsz, q_len, dim, head_dim, num_heads, num_kv_heads, past_len,
                 (half*)key_cache, (half*)value_cache,
                 nullptr, nullptr, 0, nullptr, nullptr, 0, nullptr, nullptr, 0, nullptr,
                 max_seq_len, device);
}

void ref_q4_attn_2(void* x, void* attn_output, void* o_proj, int height)
{ q4_attn_2_cuda(&g_tuning, handle(), (half*)x, (half*)attn_output, (Q4Matrix*)o_proj, height, nullptr, nullptr, 0, nullptr); }

void ref_q4_mlp(void* x, const void* rms_w, float eps, void* gate, void* up, void* down,
                int height, int dim, int device)
{
    q4_mlp_cuda(&g_tuning, (half*)x, (const half*)rms_w, eps, (Q4Matrix*)gate, (Q4Matrix*)up, (Q4Matrix*)down,
                height, dim, nullptr, nullptr, 0, nullptr, nullptr, 0, nullptr, nullptr, 0, nullptr, handle(), device);
}

int ref_sync() { return (int)cudaDeviceSynchronize(); }

// Back-to-back launches of the reference decode kernel over a pool of matrices, timed with CUDA events on the
// legacy default stream (what the reference launches on).  Returns mean microseconds per q4_matmul call.
float ref_bench_q4_pool(const void* x, int M, void** handles, int n, void* out, int reps, int mode)
{
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    for (int i = 0; i < n; i++) ref_q4_matmul(x, M, handles[i], out, 0, mode);
    cudaDeviceSynchronize();
    cudaEventRecord(a, 0);
    for (int r = 0; r < reps; r++)
        for (int i = 0; i < n; i++) ref_q4_matmul(x, M, handles[i], out, 0, mode);
    cudaEventRecord(b, 0);
    cudaEventSynchronize(b);
    float ms = 0.f; cudaEventElapsedTime(&ms, a, b);
    cudaEventDestroy(a); cudaEventDestroy(b);
    return ms * 1000.0f / (float)(reps * n);
}

}
