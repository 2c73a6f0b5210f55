/*
 * exl_b200.h -- C ABI of libexl_b200.so: the H100 (sm_90a) implementation of the
 * exllama_ext operator surface (GPTQ 4-bit matmul + the fused Llama ops around it).
 *
 * Drop-in boundary.  The reference binds this path as a torch C++ extension
 * (pybind11 module `exllama_ext`, exllama_ext/exllama_ext.cpp:743-762,
 * loaded by cuda_ext.py:43-64).  Every entry point below is what one of those 16
 * pybind functions needs underneath once the torch::Tensor arguments are
 * reduced to raw pointers and sizes; the citation on each declaration is the
 * reference function it replaces.  exllama_b200/csrc/pybind_shim.cpp is the
 * reference-side binding (same 16 names, same signatures); INTEGRATION.md shows it.
 *
 * Conventions
 *  - plain C: pointers, ints, floats.  No torch / C++ types.
 *  - all `half` data is IEEE binary16, passed as void*.
 *  - device pointers unless the name says `_host`.
 *  - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 *    The reference launches on the legacy default stream; the shim passes
 *    at::cuda::getCurrentCUDAStream().
 *  - return value: 0 on success, non-zero error code otherwise;
 *    exl_last_error() returns a human-readable message for the calling thread.
 *  - like the reference, the library keeps global per-process state (tuning,
 *    per-device scratch, handle list) and is not re-entrant across host threads.
 *  - there is NO CPU fallback anywhere: if no sm_90 device is present the
 *    compute entry points fail with EXL_ERR_CUDA.
 */
#ifndef EXL_B200_H
#define EXL_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EXL_OK            0
#define EXL_ERR_ARG       1   /* bad shape / unsupported configuration */
#define EXL_ERR_CUDA      2   /* CUDA runtime / launch error */
#define EXL_ERR_STATE     3   /* missing prepare_buffers / bad handle */

#define EXL_MAX_DEVICES   16  /* cuda_buffers.cuh:9 */

typedef struct exl_q4_matrix exl_q4_matrix;   /* opaque; reference: class Q4Matrix, q4_matrix.cuh:8-46 */

const char* exl_last_error(void);
int exl_version(void);

/* --- tuning / buffers ------------------------------------------------------ */

/* exllama_ext.cpp:89-112 set_tuning_params.  The *_no_half2 and concurrent_streams
   flags are accepted and stored for API compatibility; the sm_90a kernels have a
   single code path (fp32 accumulation) and fuse what concurrent_streams overlapped. */
int exl_set_tuning_params(int matmul_recons_thd, int fused_mlp_thd, int sdp_thd, int matmul_fused_remap,
                          int rmsnorm_no_half2, int rope_no_half2, int matmul_no_half2, int silu_no_half2,
                          int concurrent_streams);

/* exllama_ext.cpp:126-152 prepare_buffers / cuda_buffers.cu:66-89.  Borrowed scratch:
   temp_state half[temp_state_numel], temp_mlp half[temp_mlp_numel], temp_zeros_float float[max_zeros_float],
   temp_dq half[temp_dq_numel].  (The reference passes no size for temp_mlp/temp_dq; pass 0 for "unknown".) */
int exl_prepare_buffers(int device, void* temp_state, int64_t temp_state_numel,
                        void* temp_mlp, int64_t temp_mlp_numel,
                        void* temp_zeros_float, int max_zeros_float,
                        void* temp_dq, int64_t temp_dq_numel);

/* exllama_ext.cpp:117-121 cleanup: frees every Q4 handle and per-device scratch. */
int exl_cleanup(void);

/* --- Q4 matrix --------------------------------------------------------------- */

/* exllama_ext.cpp:157-194 make_q4 + q4_matrix.cu:26-53,104-168.
   qweight int32 [K/8, N], qzeros int32 [groups, N/8], scales half [groups, N] are BORROWED device memory.
   g_idx_host: int32 [K] on the host, or NULL.  When given, the rows of qweight are re-ordered by group
   IN PLACE in the caller's buffer (as the reference does) and the library keeps x_map[K] on the device. */
int exl_make_q4(void* qweight, void* qzeros, void* scales, const int32_t* g_idx_host,
                int K, int N, int groups, int device, void* stream, exl_q4_matrix** out_handle);

int exl_q4_info(const exl_q4_matrix* w, int* K, int* N, int* groups, int* groupsize, int* has_x_map, int* device);
/* copies the device x_map (uint32 [K]) to the host; for tests */
int exl_q4_get_x_map_host(const exl_q4_matrix* w, uint32_t* out_host);

/* exllama_ext.cpp:199-240 q4_matmul: out[M,N] (=|+=) x[M,K] . W.  no_zero != 0 accumulates into out
   (q4_matmul.cu:78-82).  Dispatch: skinny-M fused unpack+GEMV kernel for M <= EXL_SKINNY_MAX_M, tensor-core
   (wgmma) fused-dequant GEMM above. force_path: 0 auto, 1 skinny, 2 tensor-core GEMM, 3 reconstruct+cuBLAS. */
int exl_q4_matmul(const void* x, int M, const exl_q4_matrix* w, void* out, int no_zero, int force_path, void* stream);

/* q4_matrix.cu:212-223 Q4Matrix::reconstruct: out half [K, N] = dequantised W (bit-exact with the reference). */
int exl_q4_reconstruct(const exl_q4_matrix* w, void* out, void* stream);

/* exllama_ext.cpp:245-324 q4_matmul_lora: out = (x.A).B + x.W;  lora_temp half [M, rank]. */
int exl_q4_matmul_lora(const void* x, int M, const exl_q4_matrix* w, void* out,
                       const void* lora_A, const void* lora_B, int rank, void* lora_temp, void* stream);

/* exllama_ext.cpp:328-355 column_remap: x_new[m,i] = x[m, x_map[i]] */
int exl_column_remap(const void* x, void* x_new, int M, int K, const uint32_t* x_map, void* stream);

/* --- fp16 matmul ------------------------------------------------------------- */

/* exllama_ext.cpp:359-386 half_matmul (custom kernel; the reference requires a pre-zeroed out and
   accumulates, half_matmul.cu:15-54): out[M,N] += x[M,K] . w[K,N] */
int exl_half_matmul(const void* x, const void* w, void* out, int M, int K, int N, void* stream);
/* exllama_ext.cpp:390-420 half_matmul_cublas: out = x.w (no_zero: out += x.w), half_matmul.cu:83-125 */
int exl_half_matmul_cublas(const void* x, const void* w, void* out, int M, int K, int N, int no_zero, void* stream);

/* --- small fused ops --------------------------------------------------------- */

/* exllama_ext.cpp:606-641 rms_norm / rms_norm.cu:178-213. out may alias x. */
int exl_rms_norm(const void* x, const void* w, void* out, float epsilon, int rows, int dim, int device, void* stream);

/* exllama_ext.cpp:645-678 rope_ / rope.cu:100-125, in place.
   x half [bsz, rows_per_batch, head_dim], sin/cos half [max_seq, head_dim]. */
int exl_rope(void* x, const void* sin, const void* cos, int bsz, int rows_per_batch, int head_dim,
             int num_heads, int past_len, void* stream);

/* q4_mlp.cu:46-88 silu_mul: x = silu(x) * y, elementwise over [height, width] */
int exl_silu_mul(void* x, const void* y, int height, int width, void* stream);

/* q4_attn.cu:19-72 update_cache: cache[h, past_len + t, :] = states[t, h, :] */
int exl_update_cache(const void* key_states, const void* value_states, void* key_cache, void* value_cache,
                     int head_dim, int num_kv_heads, int q_len, int max_seq_len, int past_len, void* stream);

/* --- fused decoder blocks (decode path) --------------------------------------- */

/* exllama_ext.cpp:424-509 q4_attn / q4_attn.cu:74-204:
   rms_norm(x) -> q,k,v projections -> RoPE(q,k) -> write k,v into the cache at past_len.
   LoRA pointers may be NULL (rank 0). */
int exl_q4_attn(void* x, const void* rms_norm_weight, float epsilon,
                void* query_states, void* key_states, void* value_states,
                const exl_q4_matrix* q_proj, const exl_q4_matrix* k_proj, const exl_q4_matrix* v_proj,
                const void* sin, const void* cos,
                int bsz, int q_len, int dim, int head_dim, int num_heads, int num_kv_heads, int past_len,
                void* key_cache, void* value_cache, int max_seq_len,
                const void* q_a, const void* q_b, int q_rank,
                const void* k_a, const void* k_b, int k_rank,
                const void* v_a, const void* v_b, int v_rank,
                void* lora_temp, int device, void* stream);

/* exllama_ext.cpp:511-542 q4_attn_2 / q4_attn.cu:206-228: x += attn_output . o_proj (+ LoRA) */
int exl_q4_attn_2(void* x, const void* attn_output, const exl_q4_matrix* o_proj, int height,
                  const void* o_a, const void* o_b, int o_rank, void* lora_temp, void* stream);

/* exllama_ext.cpp:546-602 q4_mlp / q4_mlp.cu:100-199:
   x += down( silu(gate(norm(x))) * up(norm(x)) ) */
int exl_q4_mlp(void* x, const void* rms_norm_weight, float epsilon,
               const exl_q4_matrix* gate, const exl_q4_matrix* up, const exl_q4_matrix* down,
               int height, int dim,
               const void* gate_a, const void* gate_b, int gate_rank,
               const void* up_a, const void* up_b, int up_rank,
               const void* down_a, const void* down_b, int down_rank,
               void* lora_temp, int device, void* stream);

/* --- decode attention (SURVEY.md 8f-1: the ranked-first "next" row; not part of the reference's extension) ------------ */

/* Single-query attention over the KV cache, replacing the torch ops of ExLlamaAttention.fused (model.py:372-409):
   out[h, :] = softmax(q[h] . K[kvh(h), 0:seq]^T / sqrt(head_dim)) . V[kvh(h), 0:seq]      (fp32 arithmetic, fp16 in/out)
   q, out: half [num_heads * head_dim] (one token); caches: half [num_kv_heads, max_seq_len, head_dim]; head_dim == 128.
   Ordering precondition (programmatic dependent launch): the kernel loads cache rows 0 .. seq_len-2 BEFORE it waits for
   the kernel launched immediately before it on `stream` (griddepcontrol.wait); only q and row seq_len-1 are read after
   the wait.  A preceding kernel that releases its dependents early (griddepcontrol.launch_dependents -- this library's
   GEMV kernels, i.e. exl_q4_attn / exl_q4_matmul with <= 8 rows, do) may therefore produce q and cache row seq_len-1, as
   exl_q4_attn with q_len 1 does, but must not write older cache rows: after a multi-token exl_q4_attn (q_len 2..8) put
   any other kernel or a stream synchronisation before this call.  Kernels that never release early (torch ops, copies)
   are ordered as usual. */
int exl_decode_attn(const void* q, const void* key_cache, const void* value_cache, void* out,
                    int num_heads, int num_kv_heads, int head_dim, int seq_len, int max_seq_len, void* stream);

/* Causal attention of a chunk of q_len new tokens over the KV cache, read in place (exllama_b200/csrc/prefill_attn.cu).  Replaces
   repeat_kv + the additive causal mask + scaled_dot_product_attention of ExLlamaAttention.forward (model.py:447-493, mask
   model.py:1016-1018), at any past_len.  Token t of sequence b sits at absolute position past_len + t and attends rows
   [0, past_len + t] of its cache sequence:
     out[b, t, h, :] = softmax_j(q[b, t, h] . K[b, kvh(h), j] / sqrt(128)) . V[b, kvh(h), j],  j in [0, past_len + t],
     kvh(h) = h / (num_heads / num_kv_heads)
   Layouts (fp16, contiguous):
     q           [bsz, q_len, num_heads, 128]   the q projection after rope, as prefill holds it
     out         [bsz, q_len, num_heads * 128]  o_proj's input
     key_cache / value_cache  the first of bsz consecutive sequences of a [*, num_kv_heads, max_seq_len, 128] cache (a caller may
                 pass sequence seq's slice of a larger cache)
   Preconditions: cache rows [past_len, past_len + q_len) of the bsz sequences already hold this chunk's k / v.
   Guarantees: reads only cache rows [0, past_len + q_len) of the bsz sequences (rows past them may hold anything, NaN
   included); writes only out; no programmatic dependent launch, so ordinary stream order is all it needs; no atomics, so two
   launches give bitwise equal results.  Scores, softmax and accumulators are fp32, P is rounded to fp16 for the P . V product,
   the output is rounded to fp16 once.
   EXL_ERR_ARG (the message names the value) for head_dim != 128, num_kv_heads not dividing num_heads, bsz < 1, q_len < 1,
   past_len < 0, past_len + q_len > max_seq_len, or a NULL pointer. */
int exl_prefill_attn(const void* q, const void* key_cache, const void* value_cache, void* out,
                     int bsz, int q_len, int num_heads, int num_kv_heads, int head_dim,
                     int past_len, int max_seq_len, void* stream);

/* A ragged batch: n_seq sequences, each with its own chunk length, history and cache sequence (host arrays of n_seq entries, read
   during the call; the description travels in the kernel parameters, nothing is copied to the device, so a captured graph
   replays the same call).  Tokens are packed in sequence order: sequence i owns token rows [off_i, off_i + q_len[i]),
   off_i = sum_{j<i} q_len[j], T = sum_i q_len[i].  Token t of sequence i sits at position past_len[i] + t of cache sequence
   cache_seq[i].  Requirements (else EXL_ERR_ARG naming the value): 1 <= n_seq <= EXL_RAGGED_MAX_SEQ, q_len[i] >= 1,
   past_len[i] >= 0, past_len[i] + q_len[i] <= max_seq_len, 0 <= cache_seq[i] < num_cache_seqs and no cache_seq twice. */
#define EXL_RAGGED_MAX_SEQ 64
typedef struct {
    int n_seq;
    const int* q_len;
    const int* past_len;
    const int* cache_seq;
} exl_ragged;

/* exl_prefill_attn over a ragged batch, one launch (same kernel, same math inside a tile):
     out[t, h, :] = softmax_j(q[t, h] . K[cache_seq[i], kvh(h), j] / sqrt(128)) . V[cache_seq[i], kvh(h), j],
     j in [0, past_len[i] + t - off_i]  for token row t of sequence i
   q [T, num_heads, 128] after rope; out [T, num_heads * 128] (o_proj's input); key_cache / value_cache
   [num_cache_seqs, num_kv_heads, max_seq_len, 128].  One CTA per (sequence, KV group, 64-row query tile), none for padding, the
   sequences with the most keys first.  Preconditions and guarantees as exl_prefill_attn, per sequence: rows
   [past_len[i], past_len[i] + q_len[i]) of cache sequence cache_seq[i] already hold its k / v; reads only rows
   [0, past_len[i] + q_len[i]) of the named cache sequences; writes only out.  A ragged batch of bsz equal sequences in cache
   sequences 0..bsz-1 gives bitwise exl_prefill_attn's result.  EXL_ERR_ARG also for head_dim != 128, num_kv_heads not dividing
   num_heads, or a NULL pointer. */
int exl_prefill_attn_ragged(const void* q, const void* key_cache, const void* value_cache, void* out, const exl_ragged* r,
                            int num_cache_seqs, int num_heads, int num_kv_heads, int head_dim, int max_seq_len, void* stream);

/* Rope and cache write of a ragged batch in one launch: rope q [T, num_heads, 128] and k [T, num_kv_heads, 128] in place at each
   token's position (bit-exact with exl_rope, the reference's fp16 instruction order, rope.cu:48-67), and write the roped k row and
   the v [T, num_kv_heads, 128] row of token t of sequence i into row past_len[i] + t of cache sequence cache_seq[i] of
   key_cache / value_cache [num_cache_seqs, num_kv_heads, max_seq_len, 128].  sin / cos [>= max_seq_len, 128].  Writes no other
   cache row.  EXL_ERR_ARG as exl_prefill_attn_ragged. */
int exl_rope_cache_ragged(void* q, void* k, const void* v, void* key_cache, void* value_cache, const void* sin, const void* cos,
                          const exl_ragged* r, int num_cache_seqs, int num_heads, int num_kv_heads, int head_dim,
                          int max_seq_len, void* stream);

/* --- whole decode step as ONE persistent kernel (SURVEY.md 8f-4 "host loop"; 8f-2 lm_head + final norm) ------------- */

/* Everything ExLlama.forward does for one new token of one sequence (model.py:1053-1077: per layer ExLlamaAttention.fused
   :322-417 and ExLlamaMLP.fused :238-263, then the final norm and lm_head), in one cooperative launch -- see
   exllama_b200/csrc/decode_step.cu.  The plan borrows every pointer in the descriptor (weights, norms, caches, tables);
   they must stay valid and fixed for the plan's lifetime.  Restrictions: head_dim 128, num_heads % num_kv_heads == 0
   (grouped-query attention, e.g. Llama-2 70B's 64 query heads over 8 KV heads, only with tp_world == 1; 70B g128 at ctx 1920
   measured 56.3 tok/s on one H100 80GB HBM3 at a 400 W power limit), groupsize 32 * 2^n
   (or one group), widths multiples of 128, act-order (g_idx) matrices only with tp_world == 1; anything else ->
   EXL_ERR_ARG (use the per-op entry points). */
typedef struct exl_decode_plan exl_decode_plan;
typedef struct exl_decode_desc {
    int n_layers, num_heads, head_dim, max_seq_len, vocab;
    float rms_eps;
    const exl_q4_matrix* const* mats;   /* [n_layers * 7]: q, k, v, o, gate, up, down of each layer (handles from exl_make_q4) */
    const void* const* ln1;              /* [n_layers] input_layernorm weight, half [hidden] */
    const void* const* ln2;              /* [n_layers] post_attention_layernorm weight */
    void* const* key_cache;              /* [n_layers] half [max_batch, num_kv_heads, max_seq_len, head_dim] (model.py:557-585; max_batch 1
                                            unless the plan comes from exl_decode_plan_create_batch) */
    void* const* value_cache;
    const void* sin; const void* cos;    /* half [max_seq_len, head_dim] (model.py:864-877) */
    const void* final_norm;              /* half [hidden] or NULL */
    const void* lm_head;                 /* half [vocab, hidden] (nn.Linear weight, model.py:845-846) or NULL: no head */
    /* tensor parallel (SURVEY.md 8e; 0 / 1 = single GPU): this rank's column shards of q, k, v, gate, up (num_heads = LOCAL heads) and
       row shards of o, down; norms, tables, x and the head replicated.  The row-parallel partials are exchanged over NVLink inside the same
       kernel ({value, launch-epoch} 8-byte stores into every peer's slot buffer, polled by the consumer and summed in rank order):
       no separate collective, no cross-GPU barrier. */
    int tp_rank, tp_world;
    /* KV heads (grouped-query attention: k_proj / v_proj are num_kv_heads * head_dim wide, query head h attends with KV head
       h / (num_heads / num_kv_heads), model.py:310-319); 0 = num_heads, so a zero-initialised descriptor is multi-head attention */
    int num_kv_heads;
} exl_decode_desc;

int exl_decode_plan_create(const exl_decode_desc* desc, exl_decode_plan** out_plan);
/* Batched decode: a plan whose steps carry 1 .. max_batch (<= 4) sequences, each at its own context, through the same weight
   stream.  The caches hold max_batch sequences ([max_batch, num_kv_heads, max_seq_len, head_dim], ExLlamaCache(batch_size=...),
   model.py:559-577).  Not with act-order matrices or tensor parallelism; max_batch must fit the model (shared memory, and
   max_batch * num_heads -- num_kv_heads under grouped-query attention -- <= SMs); otherwise EXL_ERR_ARG naming what fits.
   exl_decode_plan_create(d, out) is exl_decode_plan_create_batch(d, 1, out). */
int exl_decode_plan_create_batch(const exl_decode_desc* desc, int max_batch, exl_decode_plan** out_plan);
/* LoRA adapters (model.py's `lora` argument, lora.py): each of the 7 projections of each layer may carry an adapter; the step adds
   (x . A) . B to that projection's output, as exl_q4_matmul_lora does, with x . A rounded to fp16 (the reference's lora_temp) and the
   product with B accumulated in fp32 into the projection (the reference's second fp16 rounding, of (x . A) . B, is skipped).  Works in
   every single-GPU configuration exl_decode_plan_create_batch accepts (multi-head and grouped-query attention, 1 .. max_batch
   sequences with the same adapter, act-order at max_batch 1).  A and B are borrowed like every other pointer of the plan; another
   adapter needs another plan.  lora == NULL or every rank 0 gives exactly exl_decode_plan_create_batch's plan.  EXL_ERR_ARG (naming the
   per-op path) for: tp_world > 1, a rank that is not a multiple of 8 in 8 .. 128, A or B not 16-byte aligned, n_layers != desc's, a
   rank > 0 with a NULL A or B. */
typedef struct exl_decode_lora {
    int n_layers;                 /* must equal desc->n_layers */
    const void* const* a;         /* [n_layers * 7] half [K, rank] (lora.py layout: A transposed) or NULL */
    const void* const* b;         /* [n_layers * 7] half [rank, N], already scaled by alpha / rank, or NULL */
    const int* rank;              /* [n_layers * 7], host; 0 = no adapter on that projection */
} exl_decode_lora;
int exl_decode_plan_create_lora(const exl_decode_desc* desc, int max_batch, const exl_decode_lora* lora, exl_decode_plan** out_plan);
int exl_decode_plan_destroy(exl_decode_plan* plan);
/* Tensor parallel set-up: export this rank's 64-byte cudaIpc handle, exchange (e.g. through torch.distributed), import all of
   them (world x 64 bytes in rank order) on every rank before the first exl_decode_step; every rank must then call
   exl_decode_step for the same token at about the same time (a rank that waits longer than 4 s for its peers traps). */
int exl_decode_plan_ipc_export(exl_decode_plan* plan, void* handle64);
int exl_decode_plan_ipc_import(exl_decode_plan* plan, const void* handles, int world);
int exl_decode_plan_info(const exl_decode_plan* plan, int* grid, int* ring_stages, int64_t* smem_bytes, int64_t* barriers_per_step);

/* Bring-up aid: with EXL_DS_TRACE=1 in the environment when the plan is created, every CTA stamps %globaltimer at its phase
   boundaries of the first 4 layers; this copies the [grid][4][24] stamps of the last launch to the host. */
int exl_decode_plan_trace(exl_decode_plan* plan, unsigned long long* out_host, int64_t capacity);

/* One token: x_in half [hidden] (the embedding row), attends over cache rows [0, past_len) plus the new row, which it
   writes at past_len.  x_out (optional) receives the final hidden state before the final norm, logits float [vocab]
   (required iff the plan has an lm_head).  CUDA-graph capturable; successive calls need no host synchronisation. */
int exl_decode_step(exl_decode_plan* plan, const void* x_in, int past_len, void* x_out, void* logits, void* stream);
/* One token for each of bsz (1 .. the plan's max_batch) sequences: x_in half [bsz][hidden]; sequence b attends over rows
   [0, past_len_host[b]) of cache sequence b and writes its new row there (sequences >= bsz are not touched); x_out half
   [bsz][hidden], logits float [bsz][vocab].  The past_len values are read on the host (baked into a CUDA-graph capture).
   exl_decode_step is this call with bsz 1 on sequence 0. */
int exl_decode_step_batch(exl_decode_plan* plan, const void* x_in, int bsz, const int* past_len_host, void* x_out, void* logits,
                          void* stream);

/* Multi-token steps: a plan whose launches carry 1 .. max_tokens (<= 4) consecutive tokens of ONE sequence -- a speculative draft
   to verify, or a short chunk such as a follow-up turn's first tokens -- in one pass over the weights; the history's K/V rows are
   read once for all of them.  The caches are [cache_seqs, num_kv_heads, max_seq_len, head_dim].  EXL_ERR_ARG for max_tokens outside
   1..4 or more than fit this model (the message names the largest that fits), act-order matrices, tp_world > 1, cache_seqs < 1.
   A multi-token plan is stepped by exl_decode_step_multi only; exl_decode_step / exl_decode_step_batch reject it. */
int exl_decode_plan_create_multi(const exl_decode_desc* desc, int max_tokens, int cache_seqs, exl_decode_plan** out_plan);
/* n (1 .. max_tokens) tokens x_in half [n][hidden] of cache sequence seq: token t sits at position past_len + t, attends cache rows
   [0, past_len) and the launch's own tokens 0 .. t, and writes row past_len + t; no other row is written, and no row at or past
   past_len is read (a speculative caller that accepts a < n tokens starts its next step at past_len + a + 1 over the stale rows).
   x_out (optional) half [n][hidden] receives the final hidden states before the final norm, logits float [n][vocab] every row
   (required iff the plan has an lm_head).  n, seq and past_len are read on the host (baked into a CUDA-graph capture).
   EXL_ERR_ARG for n outside 1..max_tokens, seq outside [0, cache_seqs), past_len < 0 or past_len + n > max_seq_len, a NULL x_in, a
   NULL logits with a head, and a plan not made by exl_decode_plan_create_multi. */
int exl_decode_step_multi(exl_decode_plan* plan, const void* x_in, int n, int seq, int past_len, void* x_out, void* logits,
                          void* stream);

/* --- tensor-parallel variants (new functionality; the reference has no tensor parallelism, SURVEY.md 8e) ----- */

/* As exl_q4_attn_2 / exl_q4_mlp, but with add_residual == 0 the row-parallel projection OVERWRITES x with this rank's
   partial product instead of accumulating into it, so that one in-place all-reduce over the ranks (rank 0 keeps the
   residual) yields x_old + sum(partials) everywhere. */
int exl_q4_attn_2_tp(void* x, const void* attn_output, const exl_q4_matrix* o_proj, int height, int add_residual, void* stream);
int exl_q4_mlp_tp(void* x, const void* rms_norm_weight, float epsilon,
                  const exl_q4_matrix* gate, const exl_q4_matrix* up, const exl_q4_matrix* down,
                  int height, int dim, int add_residual, int device, void* stream);

/* Fused projection + all-reduce over NVLink peer memory (one kernel: the GEMV epilogue pushes its tile into every peer's
   receive slot, flags it, and sums the partials of all ranks in rank order -- no NCCL call, CUDA-graph capturable).
   Setup, once per process and device: every rank allocates a workspace and exports it through cudaIpc, the 64-byte
   handles are exchanged by the host (any transport), peers are opened, then exl_tp_init installs the pointer table. */
int exl_tp_workspace_alloc(int device, void** local_ptr, void* ipc_handle_64bytes);
int exl_tp_workspace_open(int device, const void* ipc_handle_64bytes, void** peer_ptr);
int exl_tp_init(int device, int rank, int world, void* const* workspace_ptrs /* [world], own entry = local_ptr */);

/* Number of flag waits of the fused all-reduce that gave up (bounded spin) since the workspace was allocated; 0 = healthy. */
int exl_tp_status(int device, unsigned* timeouts);
/* x += all_reduce_sum(attn_output_local . o_proj_rowshard)            (every rank ends with the same x) */
int exl_q4_attn_2_ar(void* x, const void* attn_output, const exl_q4_matrix* o_proj, int height, void* stream);
/* x += all_reduce_sum(down_rowshard(silu(gate(n)) * up(n))),  n = rms_norm(x)   */
int exl_q4_mlp_ar(void* x, const void* rms_norm_weight, float epsilon,
                  const exl_q4_matrix* gate, const exl_q4_matrix* up, const exl_q4_matrix* down,
                  int height, int dim, int device, void* stream);

/* --- sampling helper (CPU, like the reference) --------------------------------- */

/* cpu_func/rep_penalty.cpp:5-31 */
int exl_rep_penalty(int vocab_size, const uint64_t* sequence_host, float* rep_mask_host,
                    float penalty_max, int sustain, int decay, int seq_len);
/* cpu_func/rep_penalty.cpp:36-74 (one batch row) */
int exl_apply_rep_penalty(int vocab_size, const uint64_t* sequence_host, float penalty_max,
                          int sustain, int decay, int seq_len, float* logits_host);

/* --- sampling on the device (exllama_b200/csrc/sample.cu; the reference samples on the host, generator.py:91-170) ---------- */

/* Settings of one exl_sample call, shared by every row (ExLlamaGenerator.Settings, generator.py:9-19). */
typedef struct {
    float temperature;        /* finite and > 0 (generator.py:106); greedy is top_k = 1 */
    int   top_k;              /* 0: off (the full order, generator.py:112-113); 1 .. vocab */
    float top_p;              /* 0: off; the loop of generator.py:120-133, including its min_p test */
    float min_p;              /* used only inside the top-p loop, as the reference does */
    float typical;            /* 0: off; generator.py:137-158, epsilon 1e-10 */
    float rep_penalty_max;    /* apply_rep_penalty_cpu semantics (cpu_func/rep_penalty.cpp:36-74); 1.0 or history == NULL: no penalty */
    int   rep_sustain;        /* -1: the whole history */
    int   rep_decay;
    int   bos_token_id;       /* >= 0: its logit becomes -10000 after the penalty (generator.py:355); -1: untouched */
    const int* banned;        /* device, n_banned ids set to -inf before the temperature (disallow_tokens, generator.py:101-102) */
    int   n_banned;
} exl_sample_params;

/* One token per row from fp32 logits [bsz][logits_ld] (read only; the reference edits its logits in place, this does not).
   Per row, in the generator's order:
     1. the repetition penalty over history[b][0 .. hist_len_host[b]) (int64 token ids, newest last), bit-exact with
        exl_apply_rep_penalty on that row: the newest occurrence of a token decides its factor, the factor steps by dv in fp32
        one position at a time;
     2. the bos logit -> -10000, then the banned logits -> -inf;
     3. / temperature (IEEE division), + 1e-8, softmax;
     4. top-k, then L1 normalisation (eps 1e-12);
     5. the top-p loop: the first token of the order is always kept, a later one while the cumulative sum that includes it is
        <= top_p and its probability >= min_p; renormalise;
     6. typical: order by |sum p log(p + 1e-10) - log(p + 1e-10)| ascending, keep the same cumulative prefix (no min_p), renormalise;
     7. the draw: the smallest kept id whose inclusive cumulative probability, in ascending token-id order, exceeds u[b]; if
        rounding leaves u[b] at or above the total, the largest kept id.
   The orders of 4-6 are probability descending and entropy deviation ascending; a tie goes to the lower token id.
   Outputs: tokens[b] (int64), probs[b] = the final probability of that token (what sample() returns), and, when dist != NULL,
   dist[b][vocab] = the final distribution (0 outside the kept set).  A row whose distribution is undefined (every logit -inf after
   masking, a NaN logit, a history or banned id outside [0, vocab)) gets token -1, probability NaN and a NaN dist row; the other
   rows are unaffected.  hist_len_host is read on the host (baked into a CUDA-graph capture).  No allocation, no floating-point
   atomics: two launches are bitwise equal.
   EXL_ERR_ARG (naming the value) for bsz outside 1 .. EXL_RAGGED_MAX_SEQ, vocab outside 1 .. 262144, logits_ld < vocab, a
   temperature that is not finite and positive, top_k outside 0 .. vocab, a negative top_p / min_p / typical, rep_sustain < -1,
   rep_decay < 0, hist_len_host[b] outside 0 .. hist_ld, or a NULL pointer (params, logits, u, tokens, probs). */
int exl_sample(const float* logits, int bsz, int vocab, int64_t logits_ld,
               const int64_t* history, int64_t hist_ld, const int* hist_len_host,
               const exl_sample_params* p, const float* u, int64_t* tokens, float* probs, float* dist, void* stream);

/* exl_sample with one parameter set per row: row b uses p_rows[b] (host array of bsz entries, read during the call and carried in the
   kernel parameters, so a captured graph replays the same call) -- its temperature, filters, penalty triple, bos id and banned list.
   Everything else is exl_sample's, and exl_sample(..., p, ...) is this call with every p_rows[b] = *p, bitwise.  EXL_ERR_ARG as
   exl_sample; a bad parameter set is reported with its row ("sample: row 3: top_k 0 ..."). */
int exl_sample_rows(const float* logits, int bsz, int vocab, int64_t logits_ld,
                    const int64_t* history, int64_t hist_ld, const int* hist_len_host,
                    const exl_sample_params* p_rows, const float* u, int64_t* tokens, float* probs, float* dist, void* stream);

/* Speculative sampling (new functionality; the reference has no speculative decoding): verify k draft tokens d_1 .. d_k of one
   sequence against the target's logits so that the emitted tokens follow exactly the target's distribution (Leviathan et al.
   2023, Chen et al. 2023).
   Inputs: target_logits fp32 [k + 1][logits_ld], row j the target's logits after the prefix and d_1 .. d_j (exl_decode_step_multi
   over [last token, d_1 .. d_k]); draft_tokens int64 [k]; draft_dist fp32 [k][dist_ld], q_j = the final distribution d_j was drawn
   from (exl_sample's dist of the draft); optional history int64 [hist_len_host] (newest last); u fp32 [k + 1] uniforms in [0, 1):
   u_0 .. u_{k-1} decide the acceptances, u_k the one draw; work fp32 [k + 1][vocab], caller-provided scratch.
   The rule:
     1. p_j = row j's final distribution under p, exactly as exl_sample computes it (same kernel), with the repetition-penalty
        history history[0 .. hist_len_host) followed by d_1 .. d_j (no history: no penalty);
     2. for j = 1 .. k: accept d_j iff u_{j-1} * q_j(d_j) < p_{j-1}(d_j) (fp32 product); stop at the first rejection;
     3. d_j rejected: the correction is drawn from r = max(0, p_{j-1} - q_j) with u_k, masses in 2^-60 fixed point: the smallest id
        whose inclusive cumulative mass, in ascending id order, exceeds floor(u_k * total) (computed in double); the largest id with
        mass if rounding leaves that at or above the total; if r has no mass at all (rounding only), the same draw over p_{j-1};
     4. all k accepted: the bonus token is exl_sample's draw of p_k with u_k.
   Outputs: *n_accepted (int32) = a in 0 .. k; tokens int64 [k + 1] = d_1 .. d_a, the correction or bonus token, then -1;
   probs fp32 [k + 1] = p of each emitted token (what sample() returns), NaN after them.  Rows past the first rejection are not
   read.  A row the walk reaches that is undefined -- p_j undefined in exl_sample's sense, d_j outside [0, vocab), q_j(d_j) not
   finite and positive -- gives *n_accepted = -1, every token -1 and every probability NaN.  k and hist_len_host are read on the
   host (baked into a CUDA-graph capture).  Two launches (exl_sample over the k + 1 rows, then spec_residual_kernel); no
   allocation, no floating-point atomics: two calls are bitwise equal.
   EXL_ERR_ARG for everything exl_sample rejects (hist_len_host < 0 included), k outside 1 .. EXL_RAGGED_MAX_SEQ - 1,
   dist_ld < vocab, or a NULL draft_tokens, draft_dist, u, work, n_accepted, tokens or probs. */
int exl_spec_verify(const float* target_logits, int k, int vocab, int64_t logits_ld,
                    const int64_t* draft_tokens, const float* draft_dist, int64_t dist_ld,
                    const int64_t* history, int hist_len_host, const exl_sample_params* p, const float* u, float* work,
                    int* n_accepted, int64_t* tokens, float* probs, void* stream);

/* --- classifier-free guidance (exllama_b200/csrc/cfg.cu; the reference: example_cfg.py:69-75) ------------------------------- */

#define EXL_CFG_MAX_PAIRS 32
/* One guided pair: logits rows a and b (the prompt and the guidance prompt), the mix weight alpha, and the repetition-penalty
   triple both rows use (exl_sample_params' rep_penalty_max / rep_sustain / rep_decay). */
typedef struct { int a, b; double alpha; float rep_penalty_max; int rep_sustain, rep_decay; } exl_cfg_pair;

/* In place on fp32 logits [rows][ld], for each of the n_pairs (1 .. EXL_CFG_MAX_PAIRS) host entries of pairs_host, pair (a, b):
     1. row a penalised over history[a][0 .. hist_len_host[a]) and row b over history[b][0 .. hist_len_host[b]) with the pair's
        triple, bit-exact with exl_apply_rep_penalty (exl_sample's rule; none when rep_penalty_max == 1, history == NULL or the
        length is 0);
     2. each penalised row x': lse = m + log sum exp(x' - m) (m its maximum; exp and the sum in float64 in one fixed order), rounded
        to fp32, and l = x' - lse in fp32;
     3. w_a = (float)(1 - alpha), w_b = (float)alpha (computed in double), mixed = w_a * l_a + w_b * l_b with each product and the
        sum rounded to fp32 (no contraction), written to both row a and row b.
   Then exl_sample(_rows) of either row with no history draws the guided token (the reference's sample_current(mixed)).  If either
   row is undefined in exl_sample's sense (a NaN logit, every logit -inf, a history id outside [0, vocab) in the penalty window),
   both rows are written all-NaN, so the sampler returns -1 for both; a NaN the mix itself produces (0 * -inf) is written as is.
   Rows in no pair are not touched.  Everything host-side is read during the call (baked into a CUDA-graph capture).  One launch,
   one cluster per pair; no allocation, no floating-point atomics: two calls are bitwise equal.
   EXL_ERR_ARG (naming the value) for rows outside 1 .. EXL_RAGGED_MAX_SEQ, vocab outside 1 .. 262144, ld < vocab, n_pairs outside
   1 .. EXL_CFG_MAX_PAIRS, a pair row outside [0, rows), a == b, a row named in two pairs, a non-finite alpha, rep_sustain < -1,
   rep_decay < 0, history without hist_len_host, hist_len_host[r] outside 0 .. hist_ld, or a NULL logits or pairs_host. */
int exl_cfg_mix(float* logits, int rows, int vocab, int64_t ld, const int64_t* history, int64_t hist_ld, const int* hist_len_host,
                const exl_cfg_pair* pairs_host, int n_pairs, void* stream);

/* --- beam search (exllama_b200/csrc/beam.cu; the reference: ExLlamaGenerator.beam_search, generator.py:497-700) ------------- */

#define EXL_BEAM_EXPAND 0
#define EXL_BEAM_FIRST 1
/* scratch exl_beam_select needs for `rows` rows and `beams` beams */
#define EXL_BEAM_WORK_BYTES(rows, beams) ((int64_t)(rows) * (beams) * 8 + (int64_t)(rows) * 4)

/* Choose beams from the rows' final distributions dist fp32 [rows][dist_ld] (exl_sample's dist rows: 0 outside the kept set).
   A candidate is a (row r, token t) with dist[r][t] > 0; its score is score_host[r] + log((double)dist[r][t]) (float64;
   score_host: host array of rows window scores, the sum of the log-probabilities of each beam's window).
     EXL_BEAM_EXPAND: the best K = min(beams, #candidates) candidates under (score descending, row ascending, token ascending),
                      written in the order (row ascending, score descending, token ascending).
     EXL_BEAM_FIRST:  rows == 1; K = min(beams, #candidates) draws without replacement with u[0 .. K) (device fp32 uniforms in
                      [0, 1)): draw j takes the smallest remaining id whose inclusive cumulative mass, in ascending id order and the
                      sampler's 2^-60 fixed point, exceeds floor(u[j] * remaining total) (computed in double), or the largest
                      remaining positive id if rounding leaves that at or above the total; the draws are written sorted by id.
   Outputs (device, beams entries each): parent int32 (the row), token int64, prob fp32 (dist of that token), score float64; entries
   past K get -1 / -1 / NaN / NaN.  *count (int32) = K, or -1 when a row is undefined: it holds a NaN, negative or infinite entry, or
   no positive one (exl_sample writes a NaN row for a distribution it marks undefined); every entry is then -1 / -1 / NaN / NaN.
   work: device scratch of at least EXL_BEAM_WORK_BYTES(rows, beams) bytes, 16-byte aligned.  rows, beams, mode and score_host are
   read on the host (baked into a CUDA-graph capture).  Two launches in expand mode (one cluster per row, one merging CTA), one in
   first mode; no allocation, no floating-point atomics: two calls are bitwise equal.
   EXL_ERR_ARG (naming the value) for rows or beams outside 1 .. EXL_RAGGED_MAX_SEQ, rows != 1 in first mode, vocab outside
   1 .. 262144, dist_ld < vocab, a mode that is neither, a NaN or +inf score_host entry, work_bytes too small, a misaligned work, or
   a NULL pointer (dist, score_host, work, parent, token, prob, score, count; u in first mode). */
int exl_beam_select(const float* dist, int rows, int vocab, int64_t dist_ld, const double* score_host, int beams, int mode, const float* u,
                    void* work, int64_t work_bytes, int* parent, int64_t* token, float* prob, double* score, int* count, void* stream);

#define EXL_KV_COPY_MAX_LAYERS 128
/* Rows [row_lo, row_hi) of cache sequence src, copied to the same rows of cache sequence dst. */
typedef struct { int src, dst, row_lo, row_hi; } exl_kv_copy_pair;

/* Copy KV-cache rows between cache sequences, every layer, K and V, in one launch: for each of the n_pairs (1 .. EXL_RAGGED_MAX_SEQ)
   host entries of pairs, rows [row_lo, row_hi) of sequence src go to the same rows of sequence dst in k_caches[l] and v_caches[l]
   for l < n_layers (host arrays of device pointers to fp16 caches [num_cache_seqs][num_kv_heads][max_seq_len][head_dim], 16-byte
   aligned).  Nothing else is written.  No sequence may be both a source and a destination and no destination may appear twice, so
   the order of the copies does not matter.  An empty range copies nothing.  One CTA per (layer, K or V, KV head, pair), each a
   contiguous run copied with 16-byte loads and stores.
   EXL_ERR_ARG (naming the value) for n_layers outside 1 .. EXL_KV_COPY_MAX_LAYERS, n_pairs outside 1 .. EXL_RAGGED_MAX_SEQ,
   num_cache_seqs < 2, num_kv_heads < 1, max_seq_len < 1, head_dim not a positive multiple of 8, a sequence outside
   [0, num_cache_seqs), a range outside 0 <= row_lo <= row_hi <= max_seq_len, a sequence that is both a source and a destination
   (src == dst included), a destination named twice, or a NULL or misaligned pointer. */
int exl_kv_copy_rows(void* const* k_caches, void* const* v_caches, int n_layers, int num_cache_seqs, int num_kv_heads, int max_seq_len,
                     int head_dim, const exl_kv_copy_pair* pairs, int n_pairs, void* stream);

/* --- batched generation (exllama_b200/csrc/generate.cu; exllama_b200/generate.py schedules requests into cache slots) ------------- */

#define EXL_GEN_MAX_STOP  8   /* stop ids per slot */
#define EXL_GEN_LIVE      0   /* slot status: still generating */
#define EXL_GEN_STOPPED   1   /* the last token stored is one of the slot's stop ids (it is kept) */
#define EXL_GEN_ERROR     4   /* the sampler returned -1 for the slot's row (undefined distribution) */

/* The uniform of draw j of a request with seed s:
     U(s, j) = (z >> 40) / 2^24,  z = splitmix64 output j (0-based) of the stream seeded with s:
       x = s + (j + 1) * 0x9E3779B97F4A7C15;  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9;  x = (x ^ (x >> 27)) * 0x94D049BB133111EB;
       z = x ^ (x >> 31)                     (all mod 2^64)
   exactly representable in fp32, in [0, 1).  A request's draws depend only on its seed and its token index. */

/* The tail of one generation step, after exl_sample(_rows) drew tokens[rows] / probs[rows].  Row r belongs to cache slot
   slot_host[r] (-1: the row is ignored); it is the request's token j_host[r], appended at history position pos_host[r].  Per slot s
   (device arrays of n_slots rows): hist int64 [n_slots][hist_ld], status int32 [n_slots], stop_ids int64 [n_slots][EXL_GEN_MAX_STOP]
   (-1 pads), seeds uint64 [n_slots]; outputs x_next fp16 [n_slots][hidden], u_next fp32 [n_slots], out_tokens int64 and out_probs
   fp32 [n_slots][out_ld].  For each row whose slot's status is EXL_GEN_LIVE:
     token t in [0, vocab): hist[s][pos] = t, out_tokens[s][j] = t, out_probs[s][j] = probs[r], status[s] = EXL_GEN_STOPPED if t is
       one of stop_ids[s], x_next[s] = embed[t] (fp16 [vocab][hidden], 16-byte loads and stores), u_next[s] = U(seeds[s], j + 1);
     else (the sampler's -1): out_tokens[s][j] = -1, out_probs[s][j] = NaN, status[s] = EXL_GEN_ERROR, nothing else.
   A row whose slot is not live writes nothing: a non-zero status is sticky until the caller resets it.  One CTA per row, no atomics:
   bitwise reproducible.  slot_host, pos_host and j_host are read on the host (baked into a CUDA-graph capture).
   EXL_ERR_ARG (naming the value) for rows outside 1 .. EXL_RAGGED_MAX_SEQ, n_slots outside 1 .. EXL_RAGGED_MAX_SEQ, a slot outside
   [-1, n_slots) or named twice, pos outside [0, hist_ld), j outside [0, out_ld), vocab < 1, hidden not a positive multiple of 8, a
   NULL or (embed, x_next) non-16-byte-aligned pointer. */
int exl_gen_advance(const int64_t* tokens, const float* probs, int rows, const int* slot_host, const int* pos_host, const int* j_host,
                    int64_t* hist, int64_t hist_ld, int* status, const int64_t* stop_ids, const uint64_t* seeds, int n_slots,
                    const void* embed, int vocab, int hidden, void* x_next, float* u_next, int64_t* out_tokens, float* out_probs,
                    int64_t out_ld, void* stream);

/* --- log-probabilities of generated tokens (exllama_b200/csrc/toplp.cu) ------------------------------------------------------ */

#define EXL_TOPLP_MAX 20   /* largest n_top of exl_top_logprobs */

/* The model's log-probabilities at each row of fp32 logits [rows][logits_ld] (1 .. EXL_RAGGED_MAX_SEQ rows, vocab 1 .. 262144): the
   row exactly as exl_sample(_rows) reads it (for a guided row, what exl_cfg_mix wrote), with no penalty, temperature, bos mask,
   banned list or filter applied -- the model's distribution, not the sampling distribution.
   A row x is undefined if it holds a NaN or a +inf, or no finite entry.  Otherwise, with m = its largest finite entry,
     S = sum over the finite entries of exp((double)x_i - m), in float64 in one fixed order;  lse = m + log(S) in float64;
     logprob(i) = (float)((double)x_i - lse)                    (-inf for a -inf logit).
   Outputs of a row (output row o, below):
     lp[o]               logprob(tokens[r]) (tokens: device int64 [rows], e.g. the sampler's draws); NaN for a token outside
                         [0, vocab) -- the sampler's -1 included -- for tokens == NULL, and for an undefined row;
     top_ids[o][i], top_lp[o][i] for i < n_top (0 .. EXL_TOPLP_MAX; row stride top_ld >= n_top): the n_top finite entries with the
                         largest logits in descending order, a tie to the lower id.  The order is on the logit itself (its bits under
                         the sign flip, -0 read as +0: an exact total order), not on exp(x - m), so underflow never ties distinct
                         logits.  Positions past the number of finite entries get id -1 and -inf; on an undefined row every id is -1
                         and every log-probability NaN.  int64 ids, fp32 log-probabilities.
   Routing: slot_host == NULL: output row o = r.  Otherwise slot_host and j_host are host arrays of rows entries, status a device
   int32 [n_slots] (exl_gen_advance's): row r writes output row o = slot_host[r] * out_ld + j_host[r] only if slot_host[r] >= 0 and
   status[slot_host[r]] == EXL_GEN_LIVE, else nothing -- exactly exl_gen_advance's gate, so a call between exl_sample_rows and
   exl_gen_advance reports the stop token too.  lp is then [n_slots][out_ld], top_ids / top_lp [n_slots][out_ld][top_ld].
   Host values are read during the call (baked into a CUDA-graph capture).  One launch, one cluster per row; no allocation, no
   floating-point atomics: two calls are bitwise equal.
   EXL_ERR_ARG (naming the value, and the row for a routing entry) for rows, vocab or n_top outside their bounds, logits_ld < vocab,
   n_top > 0 with a NULL top_ids / top_lp or top_ld < n_top, a NULL logits or lp, slot_host without j_host or status, n_slots
   outside 1 .. EXL_RAGGED_MAX_SEQ, a slot outside [-1, n_slots) or named twice, or a j outside [0, out_ld). */
int exl_top_logprobs(const float* logits, int rows, int vocab, int64_t logits_ld, const int64_t* tokens, int n_top,
                     const int* slot_host, const int* j_host, const int* status, int n_slots, int64_t out_ld,
                     float* lp, int64_t* top_ids, float* top_lp, int64_t top_ld, void* stream);

/* --- token log-probabilities (exllama_b200/csrc/logprob.cu; the reference: matmul + log_softmax + gather, perplexity.py:118-121) --- */

/* Per row t of the final-normed hidden states hn fp16 [T][H] (row-major) against lm_head fp16 [V][H] (row-major) and targets int64
   [T], with logit[t][v] = sum_k hn[t][k] * lm_head[v][k] accumulated in fp32 from exact fp16 products (never rounded to fp16, never
   written to memory):
     logprob[t] = logit[t][targets[t]] - logsumexp_v logit[t][v]   (fp32)
     greedy[t]  = argmax_v logit[t][v], ties to the lower id         (int64)
   A target outside [0, V) gives logprob NaN; a NaN or inf in row t of hn gives logprob NaN and greedy -1.  Other rows are unaffected,
   and nothing past T is written.  work: caller-provided device scratch of at least exl_token_logprobs_work_size bytes (per-row
   partials of each vocab chunk).  Two launches (the fused GEMM + per-chunk softmax statistics, then a fixed-order merge); no
   allocation, no host synchronisation and no atomics: two calls are bitwise equal, and the call can be captured in a CUDA graph.
   EXL_ERR_ARG for T < 1, V < 1, H not a positive multiple of 64, a NULL or non-16-byte-aligned pointer, work_bytes too small, or
   operands on different devices.  No GPU: EXL_ERR_CUDA (there is no CPU fallback). */
int exl_token_logprobs(const void* hn, int T, int H, const void* lm_head, int V, const int64_t* targets, float* logprob,
                       int64_t* greedy, void* work, int64_t work_bytes, void* stream);
/* *bytes = the work exl_token_logprobs needs for T rows and V ids on device `device` (it depends on the SM count). */
int exl_token_logprobs_work_size(int T, int V, int device, int64_t* bytes);

/* --- host-buffer entry point (end-to-end measurement and non-torch callers) ----- */

/* q4_matmul with HOST x / out: copies x H2D, runs exl_q4_matmul, copies out D2H, synchronises `stream`.
   x_host / out_host should be pinned for full speed.  d_x / d_out are caller-provided device staging
   buffers of M*K and M*N halves. */
int exl_q4_matmul_host(const void* x_host, int M, const exl_q4_matrix* w, void* out_host,
                       void* d_x, void* d_out, void* stream);

/* --- introspection for benchmarks ------------------------------------------------ */

/* number of kernel launches issued by this library since process start (all entry points) */
int64_t exl_launch_count(void);
/* name of the code path the last exl_q4_matmul call took ("skinny_mma", "tc_gemm", "recons_cublas") */
const char* exl_last_q4_path(void);

#define EXL_SKINNY_MAX_M 8

#ifdef __cplusplus
}
#endif
#endif /* EXL_B200_H */
