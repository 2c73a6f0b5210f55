// pybind_shim.cpp -- the reference-side binding: a torch C++ extension module named `exllama_ext` exporting
// the same 16 functions with the same signatures, argument checks and error messages as
// /root/reference/exllama_ext/exllama_ext.cpp:743-762, each one reduced to a call into the C ABI of
// libexl_b200.so (include/exl_b200.h).  model.py / generator.py of the reference run on top unchanged.
// This file contains no kernels and no arithmetic.
#include <torch/extension.h>
#include <c10/cuda/CUDAGuard.h>
#include <ATen/cuda/CUDAContext.h>
#include <cstdint>
#include <string>
#include <vector>
#include "../../include/exl_b200.h"

#define STRINGIFY_(x) #x
#define STRINGIFY(x) STRINGIFY_(x)
// same wording as exllama_ext.cpp:53-64
#define CHECK_DTYPE(x, dt) TORCH_CHECK((x).dtype() == torch::dt, #x " is incorrect datatype, must be " #dt)
#define CHECK_DTYPE_OPT(x, dt) TORCH_CHECK((x).device().is_meta() || (x).dtype() == torch::dt, #x " is incorrect datatype, must be " #dt)
#define CHECK_SHAPES(x, i, y, j, scale) TORCH_CHECK((x).size(i) == (y).size(j) * scale, #x " and " #y " have incompatible shapes")
#define CHECK_BUFFER_SIZE(buf, min) TORCH_CHECK((buf).numel() >= min, #buf " is too small")
#define CHECK_DEVICE_INDEX(idx) do { TORCH_CHECK(idx >= 0, "no device index"); TORCH_CHECK(idx < EXL_MAX_DEVICES, "invalid device index"); } while (0)
#define EXL_CALL(expr) do { int _rc = (expr); TORCH_CHECK(_rc == EXL_OK, "exl_b200: ", exl_last_error()); } while (0)

static inline void* cur_stream() { return (void*)at::cuda::getCurrentCUDAStream().stream(); }
static inline bool is_none(const torch::Tensor& t) { return t.device().is_meta(); }
static inline const void* opt_ptr(const torch::Tensor& t) { return is_none(t) ? nullptr : t.data_ptr(); }
static inline exl_q4_matrix* H(uintptr_t w) { return reinterpret_cast<exl_q4_matrix*>(w); }

void set_tuning_params(int matmul_recons_thd, int fused_mlp_thd, int sdp_thd, bool matmul_fused_remap,
                       bool rmsnorm_no_half2, bool rope_no_half2, bool matmul_no_half2, bool silu_no_half2,
                       bool concurrent_streams)
{
    EXL_CALL(exl_set_tuning_params(matmul_recons_thd, fused_mlp_thd, sdp_thd, matmul_fused_remap, rmsnorm_no_half2,
                                   rope_no_half2, matmul_no_half2, silu_no_half2, concurrent_streams));
}

void cleanup() { EXL_CALL(exl_cleanup()); }

void prepare_buffers(torch::Device device, torch::Tensor temp_state, torch::Tensor temp_mlp,
                     torch::Tensor temp_zeros_float, torch::Tensor temp_dq)
{
    int device_index = device.index();
    CHECK_DEVICE_INDEX(device_index);
    const at::cuda::OptionalCUDAGuard device_guard(device);
    EXL_CALL(exl_prepare_buffers(device_index, temp_state.data_ptr(), temp_state.numel(), temp_mlp.data_ptr(),
                                 temp_mlp.numel(), temp_zeros_float.data_ptr(), (int)temp_zeros_float.size(-1),
                                 temp_dq.data_ptr(), temp_dq.numel()));
}

uintptr_t make_q4(torch::Tensor qweight, torch::Tensor qzeros, torch::Tensor scales, torch::Tensor g_idx, int device)
{
    CHECK_DTYPE(qweight, kInt);
    CHECK_DTYPE(qzeros, kInt);
    CHECK_DTYPE(scales, kHalf);
    CHECK_DTYPE_OPT(g_idx, kInt);
    CHECK_SHAPES(qweight, 1, qzeros, 1, 8);
    CHECK_SHAPES(scales, 1, qweight, 1, 1);
    CHECK_SHAPES(qzeros, 0, scales, 0, 1);
    TORCH_CHECK(is_none(g_idx) || g_idx.device().is_cpu(), "g_idx must be a CPU tensor");
    CHECK_DEVICE_INDEX(device);
    const int width = qweight.size(1), height = qweight.size(0) * 8, groups = qzeros.size(0);
    const at::cuda::OptionalCUDAGuard device_guard(qweight.device());
    exl_q4_matrix* m = nullptr;
    EXL_CALL(exl_make_q4(qweight.data_ptr(), qzeros.data_ptr(), scales.data_ptr(),
                         is_none(g_idx) ? nullptr : (const int32_t*)g_idx.contiguous().data_ptr(),
                         height, width, groups, device, cur_stream(), &m));
    return reinterpret_cast<uintptr_t>(m);
}

void q4_matmul(torch::Tensor x, uintptr_t w, torch::Tensor out)
{
    int K = 0;
    EXL_CALL(exl_q4_info(H(w), &K, nullptr, nullptr, nullptr, nullptr, nullptr));
    CHECK_DTYPE(x, kHalf);
    CHECK_DTYPE(out, kHalf);
    CHECK_SHAPES(x, 0, out, 0, 1);
    TORCH_CHECK(K == x.size(-1), "x and w have incompatible shapes");
    const at::cuda::OptionalCUDAGuard device_guard(device_of(x));
    EXL_CALL(exl_q4_matmul(x.data_ptr(), (int)x.size(0), H(w), out.data_ptr(), 0, 0, cur_stream()));
}

void q4_matmul_lora(torch::Tensor x, uintptr_t w, torch::Tensor out, torch::Tensor lora_A, torch::Tensor lora_B,
                    torch::Tensor lora_temp)
{
    int K = 0;
    EXL_CALL(exl_q4_info(H(w), &K, nullptr, nullptr, nullptr, nullptr, nullptr));
    TORCH_CHECK(K == x.size(-1), "x and w have incompatible shapes");
    CHECK_DTYPE(x, kHalf);
    CHECK_DTYPE(out, kHalf);
    CHECK_SHAPES(x, 0, out, 0, 1);
    CHECK_SHAPES(x, 0, lora_temp, 0, 1);
    CHECK_SHAPES(x, 1, lora_A, 0, 1);
    CHECK_SHAPES(lora_A, 1, lora_B, 0, 1);
    CHECK_SHAPES(lora_B, 1, out, 1, 1);
    const at::cuda::OptionalCUDAGuard device_guard(device_of(x));
    EXL_CALL(exl_q4_matmul_lora(x.data_ptr(), (int)x.size(0), H(w), out.data_ptr(), lora_A.data_ptr(), lora_B.data_ptr(),
                                (int)lora_A.size(1), lora_temp.data_ptr(), cur_stream()));
}

void column_remap(torch::Tensor x, torch::Tensor x_new, torch::Tensor x_map)
{
    CHECK_DTYPE(x, kHalf);
    CHECK_DTYPE(x_new, kHalf);
    CHECK_DTYPE(x_map, kInt);
    CHECK_SHAPES(x_map, 0, x, 1, 1);
    const int height = x.size(0), width = x.size(1);
    CHECK_BUFFER_SIZE(x_new, height * width);
    const at::cuda::OptionalCUDAGuard device_guard(device_of(x));
    EXL_CALL(exl_column_remap(x.data_ptr(), x_new.data_ptr(), height, width, (const uint32_t*)x_map.data_ptr(), cur_stream()));
}

void half_matmul(torch::Tensor x, torch::Tensor w, torch::Tensor out)
{
    CHECK_DTYPE(x, kHalf);
    CHECK_DTYPE(w, kHalf);
    CHECK_DTYPE(out, kHalf);
    CHECK_SHAPES(x, 1, w, 0, 1);
    const at::cuda::OptionalCUDAGuard device_guard(device_of(x));
    EXL_CALL(exl_half_matmul(x.data_ptr(), w.data_ptr(), out.data_ptr(), (int)x.size(0), (int)x.size(1), (int)w.size(1), cur_stream()));
}

void half_matmul_cublas(torch::Tensor x, torch::Tensor w, torch::Tensor out)
{
    CHECK_DTYPE(x, kHalf);
    CHECK_DTYPE(w, kHalf);
    CHECK_DTYPE(out, kHalf);
    CHECK_SHAPES(x, 1, w, 0, 1);
    const at::cuda::OptionalCUDAGuard device_guard(device_of(x));
    EXL_CALL(exl_half_matmul_cublas(x.data_ptr(), w.data_ptr(), out.data_ptr(), (int)x.size(0), (int)x.size(1), (int)w.size(1), 0, cur_stream()));
}

void q4_attn(torch::Tensor x, torch::Tensor rms_norm_weight, float epsilon, torch::Tensor query_states,
             torch::Tensor key_states, torch::Tensor value_states, uintptr_t q_proj, uintptr_t k_proj, uintptr_t v_proj,
             torch::Tensor sin, torch::Tensor cos, int q_len, int past_len, int num_heads, int num_kv_heads, int head_dim,
             torch::Tensor key_cache, torch::Tensor value_cache, int max_seq_len,
             torch::Tensor q_a, torch::Tensor q_b, torch::Tensor k_a, torch::Tensor k_b, torch::Tensor v_a, torch::Tensor v_b,
             torch::Tensor lora_temp)
{
    CHECK_DTYPE(query_states, kHalf);
    CHECK_DTYPE(key_states, kHalf);
    const int bsz = query_states.size(0), dim = query_states.size(2);
    torch::Device device = x.device();
    const int device_index = device.index();
    CHECK_DEVICE_INDEX(device_index);
    const at::cuda::OptionalCUDAGuard device_guard(device);
    const int q_rank = is_none(q_a) ? 0 : q_a.size(1), k_rank = is_none(k_a) ? 0 : k_a.size(1), v_rank = is_none(v_a) ? 0 : v_a.size(1);
    EXL_CALL(exl_q4_attn(x.data_ptr(), rms_norm_weight.data_ptr(), epsilon, query_states.data_ptr(), key_states.data_ptr(),
                         value_states.data_ptr(), H(q_proj), H(k_proj), H(v_proj), sin.data_ptr(), cos.data_ptr(),
                         bsz, q_len, dim, head_dim, num_heads, num_kv_heads, past_len, key_cache.data_ptr(),
                         value_cache.data_ptr(), max_seq_len,
                         q_rank ? q_a.data_ptr() : nullptr, q_rank ? q_b.data_ptr() : nullptr, q_rank,
                         k_rank ? k_a.data_ptr() : nullptr, k_rank ? k_b.data_ptr() : nullptr, k_rank,
                         v_rank ? v_a.data_ptr() : nullptr, v_rank ? v_b.data_ptr() : nullptr, v_rank,
                         const_cast<void*>(opt_ptr(lora_temp)), device_index, cur_stream()));
}

void q4_attn_2(torch::Tensor x, torch::Tensor attn_output, uintptr_t o_proj, torch::Tensor o_a, torch::Tensor o_b,
               torch::Tensor lora_temp)
{
    CHECK_DTYPE(x, kHalf);
    CHECK_DTYPE(attn_output, kHalf);
    const at::cuda::OptionalCUDAGuard device_guard(x.device());
    const int height = x.size(0);
    const int o_rank = is_none(o_a) ? 0 : o_a.size(1);
    EXL_CALL(exl_q4_attn_2(x.data_ptr(), attn_output.data_ptr(), H(o_proj), height, o_rank ? o_a.data_ptr() : nullptr,
                           o_rank ? o_b.data_ptr() : nullptr, o_rank, const_cast<void*>(opt_ptr(lora_temp)), cur_stream()));
}

void q4_mlp(torch::Tensor x, torch::Tensor rms_norm_weight, float epsilon, uintptr_t gate, uintptr_t up, uintptr_t down,
            torch::Tensor gate_a, torch::Tensor gate_b, torch::Tensor up_a, torch::Tensor up_b, torch::Tensor down_a,
            torch::Tensor down_b, torch::Tensor lora_temp)
{
    CHECK_DTYPE(x, kHalf);
    CHECK_DTYPE(rms_norm_weight, kHalf);
    const int height = x.size(0), dim = x.size(1);
    torch::Device device = x.device();
    const int device_index = device.index();
    CHECK_DEVICE_INDEX(device_index);
    const at::cuda::OptionalCUDAGuard device_guard(device);
    const int gate_rank = is_none(gate_a) ? 0 : gate_a.size(1), up_rank = is_none(up_a) ? 0 : up_a.size(1),
              down_rank = is_none(down_a) ? 0 : down_a.size(1);
    EXL_CALL(exl_q4_mlp(x.data_ptr(), rms_norm_weight.data_ptr(), epsilon, H(gate), H(up), H(down), height, dim,
                        gate_rank ? gate_a.data_ptr() : nullptr, gate_rank ? gate_b.data_ptr() : nullptr, gate_rank,
                        up_rank ? up_a.data_ptr() : nullptr, up_rank ? up_b.data_ptr() : nullptr, up_rank,
                        down_rank ? down_a.data_ptr() : nullptr, down_rank ? down_b.data_ptr() : nullptr, down_rank,
                        const_cast<void*>(opt_ptr(lora_temp)), device_index, cur_stream()));
}

void rms_norm(torch::Tensor x, torch::Tensor w, torch::Tensor out, float epsilon)
{
    CHECK_DTYPE(x, kHalf);
    CHECK_DTYPE(w, kHalf);
    CHECK_DTYPE(out, kHalf);
    CHECK_SHAPES(x, 1, w, 0, 1);
    CHECK_SHAPES(x, 0, out, 0, 1);
    CHECK_SHAPES(x, 1, out, 1, 1);
    torch::Device device = x.device();
    const int device_index = device.index();
    CHECK_DEVICE_INDEX(device_index);
    const at::cuda::OptionalCUDAGuard device_guard(device);
    EXL_CALL(exl_rms_norm(x.data_ptr(), w.data_ptr(), out.data_ptr(), epsilon, (int)x.size(0), (int)x.size(1), device_index, cur_stream()));
}

void rope_(torch::Tensor x, torch::Tensor sin, torch::Tensor cos, int past_len, int num_heads, int head_dim)
{
    CHECK_DTYPE(x, kHalf);
    CHECK_DTYPE(sin, kHalf);
    CHECK_DTYPE(cos, kHalf);
    TORCH_CHECK(head_dim == cos.size(-1), "cos table does not match head_dim");
    TORCH_CHECK(head_dim == sin.size(-1), "sin table does not match head_dim");
    const int bsz = x.size(0);
    const int rows_per_batch = x.numel() / head_dim / bsz;
    const at::cuda::OptionalCUDAGuard device_guard(device_of(x));
    EXL_CALL(exl_rope(x.data_ptr(), sin.data_ptr(), cos.data_ptr(), bsz, rows_per_batch, head_dim, num_heads, past_len, cur_stream()));
}

void rep_penalty(torch::Tensor sequence, torch::Tensor rep_mask, float penalty_max, int sustain, int decay)
{
    CHECK_DTYPE(sequence, kLong);
    CHECK_DTYPE(rep_mask, kFloat);
    EXL_CALL(exl_rep_penalty((int)rep_mask.size(0), (const uint64_t*)sequence.data_ptr(), (float*)rep_mask.data_ptr(),
                             penalty_max, sustain, decay, (int)sequence.size(-1)));
}

void apply_rep_penalty(torch::Tensor sequence, float penalty_max, int sustain, int decay, torch::Tensor logits)
{
    CHECK_DTYPE(sequence, kLong);
    CHECK_DTYPE(logits, kFloat);
    CHECK_SHAPES(sequence, 0, logits, 0, 1);
    const int vocab_size = logits.size(-1), bsz = sequence.size(0), seq_len = sequence.size(-1);
    for (int i = 0; i < bsz; i++)
        EXL_CALL(exl_apply_rep_penalty(vocab_size, ((const uint64_t*)sequence.data_ptr()) + (size_t)i * seq_len, penalty_max,
                                       sustain, decay, seq_len, ((float*)logits.data_ptr()) + (size_t)i * vocab_size));
}

// ---- tensor-parallel additions (not part of the reference surface) -------------------------------------------------
void q4_attn_2_tp(torch::Tensor x, torch::Tensor attn_output, uintptr_t o_proj, bool add_residual)
{
    CHECK_DTYPE(x, kHalf);
    CHECK_DTYPE(attn_output, kHalf);
    const at::cuda::OptionalCUDAGuard device_guard(x.device());
    EXL_CALL(exl_q4_attn_2_tp(x.data_ptr(), attn_output.data_ptr(), H(o_proj), (int)x.size(0), add_residual, cur_stream()));
}

void q4_mlp_tp(torch::Tensor x, torch::Tensor rms_norm_weight, float epsilon, uintptr_t gate, uintptr_t up, uintptr_t down, bool add_residual)
{
    CHECK_DTYPE(x, kHalf);
    CHECK_DTYPE(rms_norm_weight, kHalf);
    torch::Device device = x.device();
    const int device_index = device.index();
    CHECK_DEVICE_INDEX(device_index);
    const at::cuda::OptionalCUDAGuard device_guard(device);
    EXL_CALL(exl_q4_mlp_tp(x.data_ptr(), rms_norm_weight.data_ptr(), epsilon, H(gate), H(up), H(down), (int)x.size(0), (int)x.size(1),
                           add_residual, device_index, cur_stream()));
}

// decode attention over the KV cache (one token): q [1, 1, heads*hd] -> out [1, 1, heads*hd]
void decode_attn(torch::Tensor q, torch::Tensor key_cache, torch::Tensor value_cache, torch::Tensor out, int num_heads,
                 int num_kv_heads, int head_dim, int seq_len, int max_seq_len)
{
    CHECK_DTYPE(q, kHalf); CHECK_DTYPE(key_cache, kHalf); CHECK_DTYPE(value_cache, kHalf); CHECK_DTYPE(out, kHalf);
    TORCH_CHECK(q.numel() == (int64_t)num_heads * head_dim && out.numel() == q.numel(), "decode_attn handles one token");
    const at::cuda::OptionalCUDAGuard device_guard(q.device());
    EXL_CALL(exl_decode_attn(q.data_ptr(), key_cache.data_ptr(), value_cache.data_ptr(), out.data_ptr(), num_heads, num_kv_heads,
                             head_dim, seq_len, max_seq_len, cur_stream()));
}

// causal attention of a chunk over the KV cache: q [bsz, q_len, heads(*hd) ...] -> out [bsz, q_len, heads*hd]; caches are the bsz
// sequences [bsz, kv_heads, max_seq_len, hd] the chunk belongs to
void prefill_attn(torch::Tensor q, torch::Tensor key_cache, torch::Tensor value_cache, torch::Tensor out, int num_heads,
                  int num_kv_heads, int head_dim, int past_len, int max_seq_len)
{
    CHECK_DTYPE(q, kHalf); CHECK_DTYPE(key_cache, kHalf); CHECK_DTYPE(value_cache, kHalf); CHECK_DTYPE(out, kHalf);
    TORCH_CHECK(q.dim() >= 2, "prefill_attn: q must be [bsz, q_len, ...]");
    const int64_t bsz = q.size(0), q_len = q.size(1);
    const int64_t tok = (int64_t)num_heads * head_dim;
    TORCH_CHECK(q.is_contiguous() && q.numel() == bsz * q_len * tok, "prefill_attn: q must be contiguous [bsz, q_len, num_heads, head_dim]");
    TORCH_CHECK(out.is_contiguous() && out.numel() == q.numel(), "prefill_attn: out must be contiguous [bsz, q_len, num_heads * head_dim]");
    const int64_t cache = bsz * num_kv_heads * (int64_t)max_seq_len * head_dim;
    TORCH_CHECK(key_cache.is_contiguous() && value_cache.is_contiguous() && key_cache.numel() == cache && value_cache.numel() == cache,
                "prefill_attn: caches must be contiguous [bsz, num_kv_heads, max_seq_len, head_dim]");
    TORCH_CHECK(key_cache.device() == q.device() && value_cache.device() == q.device() && out.device() == q.device(),
                "prefill_attn: tensors on different devices");
    const at::cuda::OptionalCUDAGuard device_guard(q.device());
    EXL_CALL(exl_prefill_attn(q.data_ptr(), key_cache.data_ptr(), value_cache.data_ptr(), out.data_ptr(), (int)bsz, (int)q_len,
                              num_heads, num_kv_heads, head_dim, past_len, max_seq_len, cur_stream()));
}

// a ragged batch: the three per-sequence lists as exl_ragged (the vectors must outlive the call)
static exl_ragged ragged_of(const std::vector<int>& q_lens, const std::vector<int>& past_lens, const std::vector<int>& cache_seqs,
                            const char* who)
{
    TORCH_CHECK(q_lens.size() == past_lens.size() && q_lens.size() == cache_seqs.size(), who,
                ": q_lens, past_lens and cache_seqs must have the same length");
    return exl_ragged{(int)q_lens.size(), q_lens.data(), past_lens.data(), cache_seqs.data()};
}

static int64_t ragged_tokens(const std::vector<int>& q_lens)
{
    int64_t T = 0;
    for (int l : q_lens) T += l;
    return T;
}

static void check_caches(const torch::Tensor& kc, const torch::Tensor& vc, const torch::Tensor& like, int num_kv_heads, int head_dim,
                         int max_seq_len, const char* who)
{
    CHECK_DTYPE(kc, kHalf); CHECK_DTYPE(vc, kHalf);
    TORCH_CHECK(kc.dim() == 4 && kc.is_contiguous() && vc.is_contiguous() && kc.sizes() == vc.sizes() && kc.size(1) == num_kv_heads &&
                kc.size(2) == max_seq_len && kc.size(3) == head_dim,
                who, ": caches must be contiguous [num_cache_seqs, num_kv_heads, max_seq_len, head_dim]");
    TORCH_CHECK(kc.device() == like.device() && vc.device() == like.device(), who, ": tensors on different devices");
}

// causal attention of a ragged batch over the caches: q [T, heads(*hd)] packed -> out [T, heads*hd]; sequence i attends cache
// sequence cache_seqs[i] of caches [num_cache_seqs, kv_heads, max_seq_len, hd]
void prefill_attn_ragged(torch::Tensor q, torch::Tensor key_cache, torch::Tensor value_cache, torch::Tensor out,
                         std::vector<int> q_lens, std::vector<int> past_lens, std::vector<int> cache_seqs, int num_heads,
                         int num_kv_heads, int head_dim, int max_seq_len)
{
    const char* who = "prefill_attn_ragged";
    CHECK_DTYPE(q, kHalf); CHECK_DTYPE(out, kHalf);
    const exl_ragged r = ragged_of(q_lens, past_lens, cache_seqs, who);
    const int64_t n = ragged_tokens(q_lens) * num_heads * head_dim;
    TORCH_CHECK(q.is_contiguous() && q.numel() == n, who, ": q must be contiguous [sum(q_lens), num_heads, head_dim]");
    TORCH_CHECK(out.is_contiguous() && out.numel() == n, who, ": out must be contiguous [sum(q_lens), num_heads * head_dim]");
    check_caches(key_cache, value_cache, q, num_kv_heads, head_dim, max_seq_len, who);
    TORCH_CHECK(out.device() == q.device(), who, ": tensors on different devices");
    const at::cuda::OptionalCUDAGuard device_guard(q.device());
    EXL_CALL(exl_prefill_attn_ragged(q.data_ptr(), key_cache.data_ptr(), value_cache.data_ptr(), out.data_ptr(), &r,
                                     (int)key_cache.size(0), num_heads, num_kv_heads, head_dim, max_seq_len, cur_stream()));
}

// rope q [T, heads(*hd)] and k [T, kv_heads(*hd)] of a ragged batch in place and write k, v [T, kv_heads(*hd)] into the caches
void rope_cache_ragged(torch::Tensor q, torch::Tensor k, torch::Tensor v, torch::Tensor key_cache, torch::Tensor value_cache,
                       torch::Tensor sin, torch::Tensor cos, std::vector<int> q_lens, std::vector<int> past_lens,
                       std::vector<int> cache_seqs, int num_heads, int num_kv_heads, int head_dim, int max_seq_len)
{
    const char* who = "rope_cache_ragged";
    CHECK_DTYPE(q, kHalf); CHECK_DTYPE(k, kHalf); CHECK_DTYPE(v, kHalf); CHECK_DTYPE(sin, kHalf); CHECK_DTYPE(cos, kHalf);
    const exl_ragged r = ragged_of(q_lens, past_lens, cache_seqs, who);
    const int64_t T = ragged_tokens(q_lens);
    TORCH_CHECK(q.is_contiguous() && q.numel() == T * num_heads * head_dim, who, ": q must be contiguous [sum(q_lens), num_heads, head_dim]");
    TORCH_CHECK(k.is_contiguous() && v.is_contiguous() && k.numel() == T * num_kv_heads * head_dim && v.numel() == k.numel(), who,
                ": k and v must be contiguous [sum(q_lens), num_kv_heads, head_dim]");
    TORCH_CHECK(sin.is_contiguous() && cos.is_contiguous() && sin.numel() >= (int64_t)max_seq_len * head_dim &&
                cos.numel() >= (int64_t)max_seq_len * head_dim, who, ": sin and cos must be contiguous [>= max_seq_len, head_dim]");
    check_caches(key_cache, value_cache, q, num_kv_heads, head_dim, max_seq_len, who);
    TORCH_CHECK(k.device() == q.device() && v.device() == q.device() && sin.device() == q.device() && cos.device() == q.device(), who,
                ": tensors on different devices");
    const at::cuda::OptionalCUDAGuard device_guard(q.device());
    EXL_CALL(exl_rope_cache_ragged(q.data_ptr(), k.data_ptr(), v.data_ptr(), key_cache.data_ptr(), value_cache.data_ptr(),
                                   sin.data_ptr(), cos.data_ptr(), &r, (int)key_cache.size(0), num_heads, num_kv_heads, head_dim,
                                   max_seq_len, cur_stream()));
}

// fused projection + peer-memory all-reduce
pybind11::tuple tp_workspace_alloc(int device)
{
    void* p = nullptr; char h[64];
    EXL_CALL(exl_tp_workspace_alloc(device, &p, h));
    return pybind11::make_tuple(reinterpret_cast<uintptr_t>(p), pybind11::bytes(h, 64));
}
uintptr_t tp_workspace_open(int device, pybind11::bytes handle)
{
    std::string h = handle;
    TORCH_CHECK(h.size() == 64, "ipc handle must be 64 bytes");
    void* p = nullptr;
    EXL_CALL(exl_tp_workspace_open(device, h.data(), &p));
    return reinterpret_cast<uintptr_t>(p);
}
void tp_init(int device, int rank, int world, std::vector<uintptr_t> ptrs)
{
    std::vector<void*> v; for (auto p : ptrs) v.push_back(reinterpret_cast<void*>(p));
    TORCH_CHECK((int)v.size() == world, "tp_init: need one workspace pointer per rank");
    EXL_CALL(exl_tp_init(device, rank, world, v.data()));
}
void q4_attn_2_ar(torch::Tensor x, torch::Tensor attn_output, uintptr_t o_proj)
{
    CHECK_DTYPE(x, kHalf);
    CHECK_DTYPE(attn_output, kHalf);
    const at::cuda::OptionalCUDAGuard device_guard(x.device());
    EXL_CALL(exl_q4_attn_2_ar(x.data_ptr(), attn_output.data_ptr(), H(o_proj), (int)x.size(0), cur_stream()));
}
void q4_mlp_ar(torch::Tensor x, torch::Tensor rms_norm_weight, float epsilon, uintptr_t gate, uintptr_t up, uintptr_t down)
{
    CHECK_DTYPE(x, kHalf);
    CHECK_DTYPE(rms_norm_weight, kHalf);
    const int device_index = x.device().index();
    CHECK_DEVICE_INDEX(device_index);
    const at::cuda::OptionalCUDAGuard device_guard(x.device());
    EXL_CALL(exl_q4_mlp_ar(x.data_ptr(), rms_norm_weight.data_ptr(), epsilon, H(gate), H(up), H(down), (int)x.size(0), (int)x.size(1),
                           device_index, cur_stream()));
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m)
{
    m.def("set_tuning_params", &set_tuning_params, "set_tuning_params");
    m.def("prepare_buffers", &prepare_buffers, "prepare_buffers");
    m.def("cleanup", &cleanup, "cleanup");
    m.def("make_q4", &make_q4, "make_q4");
    m.def("q4_matmul", &q4_matmul, "q4_matmul");
    m.def("q4_matmul_lora", &q4_matmul_lora, "q4_matmul_lora");
    m.def("q4_attn", &q4_attn, "q4_attn");
    m.def("q4_attn_2", &q4_attn_2, "q4_attn_2");
    m.def("q4_mlp", &q4_mlp, "q4_mlp");
    m.def("column_remap", &column_remap, "column_remap");
    m.def("rms_norm", &rms_norm, "rms_norm");
    m.def("rope_", &rope_, "rope_");
    m.def("half_matmul", &half_matmul, "half_matmul");
    m.def("half_matmul_cublas", &half_matmul_cublas, "half_matmul_cublas");
    m.def("rep_penalty", &rep_penalty, "rep_penalty");
    m.def("apply_rep_penalty", &apply_rep_penalty, "apply_rep_penalty");
    // additions for tensor parallelism
    m.def("q4_attn_2_tp", &q4_attn_2_tp, "q4_attn_2_tp");
    m.def("q4_mlp_tp", &q4_mlp_tp, "q4_mlp_tp");
    m.def("decode_attn", &decode_attn, "decode_attn");
    m.def("prefill_attn", &prefill_attn, "prefill_attn");
    m.def("prefill_attn_ragged", &prefill_attn_ragged, "prefill_attn_ragged");
    m.def("rope_cache_ragged", &rope_cache_ragged, "rope_cache_ragged");
    m.def("tp_status", [](int device) { unsigned t = 0; EXL_CALL(exl_tp_status(device, &t)); return (int)t; }, "tp_status");
    m.def("tp_workspace_alloc", &tp_workspace_alloc, "tp_workspace_alloc");
    m.def("tp_workspace_open", &tp_workspace_open, "tp_workspace_open");
    m.def("tp_init", &tp_init, "tp_init");
    m.def("q4_attn_2_ar", &q4_attn_2_ar, "q4_attn_2_ar");
    m.def("q4_mlp_ar", &q4_mlp_ar, "q4_mlp_ar");
}
