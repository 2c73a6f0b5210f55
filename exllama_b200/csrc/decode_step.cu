// decode_step.cu -- ONE persistent cooperative kernel for a whole decode token (q_len 1; 1 .. 4 sequences) on sm_90a.
//
// SURVEY.md 8f-4 ("host loop: a C++ decoder_layer op / whole-step capture") and the answer to VERDICT r1 item 1: the five
// launches per layer (q4_attn, decode_attn, q4_attn_2, q4_mlp x2) were latency-bound -- launch + setup + x-dependent
// prologue + split-K exchange around 1-9 us of streaming each.  Here the whole token is one launch:
//
//   for every layer:   QKV | ATT | O | GU | DOWN        (| = grid barrier)       then  final norm + fp16 lm_head
//
// replacing, per layer, rms_norm + 3 x q4_matmul + 2 x rope + update_cache (q4_attn.cu:74-165), the torch attention ops
// (model.py:383-409), q4_matmul += residual (q4_attn.cu:206-228), rms_norm + 2 x q4_matmul + silu_mul + q4_matmul += residual
// (q4_mlp.cu:100-199), and at the end model.py:1069-1077 (norm + lm_head).
//
// Structure (one CTA per SM; 16 consumer warps + 4 producer warps = 4 pipelines of {1 producer, 4 consumer warps, own ring slice}):
//  * The PRODUCER warps walk a static schedule of 8 KB "stages" (stage j of the CTA belongs to pipeline j & 3) through a
//    shared-memory ring with full/empty mbarriers and never wait for a grid barrier: weight units (ONE 3-D TMA op for the
//    8 KB of packed qweight + one 2-D op each for the unit's scale and zero rows), KV-cache rows older than the current token
//    (bulk copies) and lm_head rows do not depend on activations, so up to 4 x depth x 8 KB per SM (~19 MB chip-wide) of the
//    NEXT phase is loaded while the consumers are in a barrier or in a phase prologue, one stage per pipeline in flight at a
//    time (up to MID_INFLIGHT later in a phase, away from the barriers).  HBM stays busy across phase and layer boundaries -- the thing separate launches could not do.
//  * Work of a GEMV phase = (128-column tile) x (128-row K stage) units, flattened tile-major and cut into G equal contiguous
//    ranges (G = grid size): every SM streams the same number of bytes whatever the matrix shapes (65B gate/up: 172 tiles on
//    132 SMs is no longer a problem).  A warp accumulates its 32 columns over the stages it sees and, at a tile boundary,
//    adds its fp32 partial into the phase's accumulator in L2 with red.global.add.v4.f32 -- the split-K reduction is the
//    grid barrier that the data dependence needs anyway.
//  * Inner product exactly as q4_gemv.cu (integer tensor cores, nibbles as the A operand straight from the ring, x carried
//    per quantisation segment as a 16-bit integer), specialised for one token: the two byte planes of x ride in two of the
//    eight B columns, so ONE mma.sync.m16n8k32.u8.s8 per 16 columns x 32 k does both planes.
//  * The x-dependent part of a phase (residual add + RMS norm, rope + cache write, softmax-combine, silu*mul; then per-segment
//    quantisation of the K range this CTA needs) runs after the barrier out of L2-resident fp32 accumulators; the residual
//    stream itself lives in every CTA's shared memory in fp16, rounded where the reference rounds it.
//  * ATT: (KV head, 16-position chunk) units, online softmax per warp in fp32 (as decode_attn.cu), partial (m, l, o) per CTA and
//    query head to L2, combined in the O prologue.  The newest K/V row never round-trips through HBM before it is used.  Under
//    grouped-query attention one 8 KB stage of K/V serves all n_rep query heads of its group: the K/V bytes are read once per KV head.
//  * HEAD: lm_head [vocab, hidden] fp16 streamed as 8 KB stages, fp32 dot products, fp32 logits by red.global.add.
//  * Batched decode (template flag BATCH, up to MAX_BATCH = 4 sequences, each at its own context): the same weight stages, ring and
//    IMMAs serve every sequence.  Sequence b's two x planes ride in B columns 2b, 2b + 1, so lane t of an MMA quad ends up holding
//    sequence t's result; ATT runs over virtual heads (sequence, head) with each sequence's own context and cache rows; the head
//    dots every lm_head stage with every sequence.  Only the K/V bytes grow with the batch.  The prologues and the head are written
//    once, as loops over the nb sequences of the launch; without BATCH nb is the compile-time 1 and the loops fold away.
//  * Multi-token steps (template flag MULTI, with BATCH and the grouped-query ATT path for any n_rep): up to 4 consecutive tokens of ONE
//    sequence (speculative verification, short chunks).  Token t sits at past_len + t; ATT runs over the real KV heads at past_len, so
//    the history's K/V bytes are read once for all tokens, each stage serving n_rep x n query vectors, and a causal tail partial over
//    the launch's own new rows 0 .. t (kept in shared memory) replaces the single new-token partial.  No row >= past_len is read.
//  * LoRA adapters (template flag LORA, one GPU): an adapted phase gets an LA step after its prologue (t = x . A over (matrix, K stage)
//    units, fp32 red.add into L2, one grid barrier), and the CTA owning K stage 0 of an adapted tile adds fp16(t) . B to it after the
//    GEMV (decode_step_sched.h: lora_*).
//
// Restrictions (checked on the host; anything else uses the per-op kernels): head_dim 128, heads % kv_heads == 0 (grouped-query
// attention only without tensor parallelism), groupsize 32 * 2^n (or one group), widths multiples of 128, act-order only without
// tensor parallelism (template flag ACT: x is gathered through
// each matrix's x_map while it is staged).  Tensor parallel (template flag TP): the row-parallel partials are exchanged by
// {value, epoch} stores into the peers' memory, see StepArgs.  Every wait is bounded by wall time and traps on expiry.
#include "exl_common.cuh"
#include "decode_step_sched.h"
#include <cstring>
#include <type_traits>
#include <vector>

namespace {

using namespace ds_sched;                        // TILE, W_BYTES, STAGE_STRIDE, PART_LD, MAX_DEPTH, PH_*, Phase, phase_of, range_lo, share_lo, cta_of

constexpr int DS_CONSUMERS = 512;                // 16 consumer warps = 4 pipelines x 4 column-warps
constexpr int DS_NCW = DS_CONSUMERS / 32;
constexpr int DS_NPW = 4;                        // producer warps, one per pipeline
constexpr int DS_THREADS = DS_CONSUMERS + 32 * DS_NPW;
constexpr int BOX_BYTES = 2048;                  // one column group of the unit: 16 k8-rows x 32 columns, SWIZZLE_128B
constexpr int META_SC = W_BYTES;                 // up to 4 group rows of 128 fp16 scales
constexpr int META_ZQ = W_BYTES + 1024;          // up to 4 group rows of 128 zero nibbles
constexpr int MAX_LAYERS = 128;
constexpr int TRACE_LAYERS = 4;
enum { ZR_QKV = 0, ZR_H = 1, ZR_GU = 2, ZR_LOGITS = 3, ZR_HALF = 4, ZR_COUNT = 5 };     // zero_share / push ranges
constexpr unsigned long long WAIT_NS = 4000000000ull;   // any single wait longer than this aborts the launch
constexpr int MID_INFLIGHT = 3;                  // ring stages in flight per pipeline past the first `depth` stages of a phase

struct alignas(64) LayerDesc
{
    CUtensorMap tw[7];                 // q k v o gate up down: exl_q4_matrix::tmap_w3 (one 8 KB unit per op)
    CUtensorMap ts[7];                 // ::tmap_sc
    CUtensorMap tz[7];                 // ::tmap_qz
    const uint32_t* xmap[7];           // act-order: x column feeding sequential row k of each matrix (exl_q4_matrix::x_map), else NULL
    const half* ln1; const half* ln2;
    half* kc; half* vc;                // [max_batch, kv_heads, max_seq, 128]
};

// one projection's LoRA adapter: A [K, rank] and B [rank, N] fp16 row-major (B already scaled by alpha / rank); rank 0 = none
struct LoraMat { const half* a; const half* b; int rank; int t_off; };

struct StepArgs
{
    const LayerDesc* layers; int n_layers;
    int H, HQ, HKV, I;                 // hidden, attention width (heads * 128), k / v width (kv_heads * 128), intermediate width
    int heads, kv_heads, n_rep;        // query heads, KV heads, query heads per KV head (1: multi-head attention)
    int max_seq, past_len;             // past_len: the longest context of the batch
    int gshift;                        // log2(groupsize / 32); 30 = one group per matrix
    int depth;                         // ring stages per pipeline (4 pipelines)
    int spt_max;                       // max K / 128 over the phases
    int act;                           // act-order matrices present: x is gathered through each matrix's x_map while it is staged; the
                                       // matrices of a phase then need their own quantised x (two staging slots), and o_proj's input
                                       // (a gather over all heads) goes through one extra combine step + barrier
    half* attn_vec;                    // [HQ] combined attention output (act-order only)
    float eps;
    const half* x_in; half* x_out;     // [bsz][H] input hidden states; final hidden states (before the final norm), optional
    const half* sin; const half* cos;  // [max_seq, 128]
    const half* final_norm; const half* lm_head; float* logits; int vocab;     // optional head; logits [bsz][vocab]
    float* acc_qkv; float* acc_o; float* acc_gu; float* acc_d;                 // fp32 phase accumulators in L2, [bsz][width] each
    float* att_part; int att_slots;    // [bsz * heads][att_slots][PART_LD] (virtual query heads)
    unsigned long long* bar;           // grid barrier: monotonic arrival counter (this GPU's CTAs only)
    // tensor parallel (world > 1): after a row-parallel projection (o_proj, down_proj) every rank's partial [H] vector -- already
    // reduced over its own CTAs in L2 -- is stored straight into slot [rank] of EVERY peer over NVLink as 8-byte {value, epoch}
    // pairs (posted writes, H / grid elements per CTA and peer).  There is no cross-GPU barrier and no system-scope fence: the next
    // prologue polls each pair until its epoch matches (an 8-byte store is single-copy atomic, as in NCCL's LL protocol), and the
    // slots cannot be overwritten early because a peer's next partial causally depends on this rank's next one.  One-shot
    // all-reduce inside the kernel: no separate collective, no host involvement, CUDA-graph replayable (the epoch comes from a
    // device-side launch counter).
    int tp_rank, tp_world;
    uint2* push_o[8]; uint2* push_d[8];          // where THIS rank's partial goes on rank r: slots_o / slots_d of rank r, row tp_rank
    const uint2* slots_o; const uint2* slots_d;  // own receive slots [world][H] of {float bits, epoch}
    unsigned* launch_ctr;                        // launches completed so far (all ranks run the same number)
    int tp_reduce;                               // world >= 4: each CTA totals ITS share of the ranks' partials after the push and a second local
                                                 // barrier publishes the complete sum (prologues then read one vector instead of world)
    int debug;                         // EXL_DS_DEBUG bitmask (bring-up experiments): 1 skip GEMV math, 2 skip attention math, 4 skip head math
    unsigned long long* trace;         // optional [G][TRACE_LAYERS][16] globaltimer stamps of CTA thread 0 (EXL_DS_TRACE=1), else NULL
    // batched decode (BATCH kernels only; the others read none of these)
    int bsz;                           // sequences of this launch, 1 .. max_batch of the plan
    int xst;                           // compacted x staging stages per sequence (decode_step_sched.h: batch_xstages)
    int past_lens[MAX_BATCH];          // context of each sequence
    // LoRA adapters (LORA kernels only; the others read none of these): [n_layers * 7] matrices' adapters, and the fp32 t = x . A
    // accumulators in L2 (matrix of rank r at t_off: [max_batch][r]), zeroed at launch start
    const LoraMat* lora; float* lora_t; int lora_t4;              // lora_t4: floats of lora_t / 4
    // multi-token steps (MULTI kernels only): the bsz tokens of the launch sit at positions past_len + t of cache sequence seq
    int seq;
};

// ------------------------------------------------------------------------------------------------------------ helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ void mbar_init(void* bar, int count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory"); }
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// NOTE on parities: a waiter may be at most ONE phase ahead of the barrier (try_wait.parity cannot tell phase k from k + 2).
// Every warp of a pipeline visits every stage of that pipeline in order, so this always holds here.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    if (mbar_try(bar, parity)) return;
    const unsigned long long t0 = gtime();
    for (unsigned i = 1; !mbar_try(bar, parity); i++)
        if ((i & 1023u) == 0 && gtime() - t0 > WAIT_NS) __trap();
}
// HBM -> shared memory through the TMA unit, completing on mbarrier `bar`; pol: L2 cache policy (createpolicy)
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t pol)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 :: "r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(pol) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tmap, int c0, int c1, uint32_t bar, uint64_t pol)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3}], [%4], %5;"
                 :: "r"(dst), "l"(tmap), "r"(c0), "r"(c1), "r"(bar), "l"(pol) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tmap, int c0, int c1, int c2, uint32_t bar, uint64_t pol)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3, %4}], [%5], %6;"
                 :: "r"(dst), "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(bar), "l"(pol) : "memory");
}
// wait that hands back a zero "token": adding it to the addresses of the loads that follow makes them data-dependent on the wait, so
// the (non-volatile, freely schedulable) shared-memory loads below can never be hoisted above it
__device__ __forceinline__ uint32_t mbar_wait_tok(uint32_t bar, uint32_t parity, bool already)
{
    if (!already) mbar_wait(bar, parity);
    uint32_t z;
    asm volatile("mov.u32 %0, 0;" : "=r"(z) :: "memory");
    return z;
}
// arrive that consumes a value computed from the stage's data: it cannot be scheduled before the loads it releases
__device__ __forceinline__ void mbar_arrive_dep(uint32_t bar, float dep)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar), "f"(dep) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t a)
{
    uint4 r; asm("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a)); return r;
}
__device__ __forceinline__ uint2 lds64(uint32_t a)
{
    uint2 r; asm("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "r"(a)); return r;
}
__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t r; asm("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(a)); return r; }
// 8-byte shared load that happens only when `on` (else zeros): a warp-uniform bound becomes a predicate instead of a branch
__device__ __forceinline__ uint2 lds64_if(uint32_t a, bool on)
{
    uint2 r = make_uint2(0u, 0u);
    asm("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %3, 0;\n\t@q ld.shared.v2.u32 {%0, %1}, [%2];\n\t}" : "+r"(r.x), "+r"(r.y) : "r"(a), "r"((uint32_t)on));
    return r;
}
// 2^x, flush-to-zero: exp(y) = ex2(y * log2 e); -inf -> 0
__device__ __forceinline__ float ex2_ftz(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 512;" ::: "memory"); }
__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d)
{
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" :: "l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }

// u8 (weights, 0..15) x s8 (x planes) -> s32; first MMA of a segment starts from C = 0
__device__ __forceinline__ void imma(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1)
{
    asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void imma_z(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1)
{
    asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
        : "=r"(c[0]), "=r"(c[1]), "=r"(c[2]), "=r"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "r"(0));
}

// acc += w.lo * x.lo + w.hi * x.hi for two packed fp16 pairs, in that order.  The product of two fp16 values is exact in fp32, so
// converting both to fp32 and fmaf() rounds once per term (sm_90 has no mixed fp16 x fp16 + fp32 FMA instruction).
__device__ __forceinline__ float fhfma2(uint32_t w, uint32_t x, float acc)
{
    const float2 wf = __half22float2(*reinterpret_cast<const half2*>(&w)), xf = __half22float2(*reinterpret_cast<const half2*>(&x));
    return fmaf(wf.y, xf.y, fmaf(wf.x, xf.x, acc));
}

__device__ __forceinline__ half silu_h(half x)
{
    // same fp16 sequence as the reference (q4_mlp.cu:27-36)
    const half one = __float2half(1.0f);
    const half e = hexp(__hneg(x));
    const half r = hrcp(__hadd(one, e));
    return __hmul(x, r);
}

// One k8-row (8 halves) -> 16-bit integers x_q = 256 a + b with BOTH bytes signed (b = sign-extended low byte,
// a = (x_q + 128) >> 8), packed {a(0,2,4,6), a(1,3,5,7), b(0,2,4,6), b(1,3,5,7)}; returns sum of x_q.  |x_q| <= 32639 keeps a in s8.
__device__ __forceinline__ int quantise_row(const uint4& hv, float inv, uint4& o)
{
    const half2* h = reinterpret_cast<const half2*>(&hv);
    int sum = 0;
    o = make_uint4(0, 0, 0, 0);
    #pragma unroll
    for (int i = 0; i < 4; i++) {
        const float2 f = __half22float2(h[i]);
        const int q0 = __float2int_rn(f.x * inv), q1 = __float2int_rn(f.y * inv);
        sum += q0 + q1;
        o.x |= (uint32_t)(((q0 + 128) >> 8) & 0xff) << (8 * i);
        o.y |= (uint32_t)(((q1 + 128) >> 8) & 0xff) << (8 * i);
        o.z |= (uint32_t)(q0 & 0xff) << (8 * i);
        o.w |= (uint32_t)(q1 & 0xff) << (8 * i);
    }
    return sum;
}
// the 8 x columns feeding k8-row k8 of an act-order matrix (identity when the matrix has no x_map)
__device__ __forceinline__ void load_map8(const uint32_t* map, int k8, uint32_t (&idx)[8])
{
    if (map) {
        const uint4 m0 = __ldg(reinterpret_cast<const uint4*>(map) + 2 * k8), m1 = __ldg(reinterpret_cast<const uint4*>(map) + 2 * k8 + 1);
        idx[0] = m0.x; idx[1] = m0.y; idx[2] = m0.z; idx[3] = m0.w; idx[4] = m1.x; idx[5] = m1.y; idx[6] = m1.z; idx[7] = m1.w;
    } else {
        #pragma unroll
        for (int i = 0; i < 8; i++) idx[i] = (uint32_t)(k8 * 8 + i);
    }
}
__device__ __forceinline__ float row_absmax(const uint4& hv)
{
    const half2* h = reinterpret_cast<const half2*>(&hv);
    float mx = 0.f;
    #pragma unroll
    for (int i = 0; i < 4; i++) { const float2 f = __half22float2(__habs2(h[i])); mx = fmaxf(mx, fmaxf(f.x, f.y)); }
    return mx;
}

// Grid-wide barrier for the consumer threads of all CTAs: one monotonic 64-bit arrival counter (never reset, so graph replays
// and back-to-back launches need no host-side state); every CTA adds 1 with release semantics and polls until the count reaches
// the target of this barrier.  One L2 round trip to arrive, one to observe.
__device__ __forceinline__ void grid_barrier(unsigned long long* ctr, unsigned long long& target, unsigned nctas, int tid,
                                             volatile int* arrived = nullptr)
{
    consumer_sync();
    if (tid == 0) {
        asm volatile("red.release.gpu.global.add.u64 [%0], 1;" :: "l"(ctr) : "memory");
        if (arrived) *arrived = *arrived + 1;
        unsigned long long v;
        asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(ctr) : "memory");
        if (v < target) {
            const unsigned long long t0 = gtime();
            unsigned i = 0;
            do {
                asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(ctr) : "memory");
                if ((++i & 1023u) == 0 && gtime() - t0 > WAIT_NS) __trap();
            } while (v < target);
        }
    }
    target += nctas;
    consumer_sync();
}

// ACT: act-order matrices present; TP: tensor parallel; GQA: grouped-query attention (kv_heads < heads, single GPU); BATCH: a plan
// for more than one sequence (neither ACT nor TP).  Compile-time so that the common kernel (none of them) carries none of their
// address arithmetic, branches or code (the runtime-flag version of the same source was 10 % slower on the plain 7B step; a runtime
// n_rep branch around the attention phase made ptxas spill in it).  Without BATCH, nb below is the constant 1.  LORA: a plan with
// LoRA adapters (single GPU; any of the others but TP): the LA steps and B terms below.  MULTI: bsz consecutive tokens of ONE sequence
// (with BATCH and GQA, for any n_rep; neither ACT, TP nor LORA): the batch's GEMV, norm and head phases, and ATT over the real KV
// heads at the shared context past_len, each stage serving n_rep * bsz query vectors, plus a causal tail over the launch's own rows.
template <bool MULTI> __device__ __forceinline__ Phase step_phase(const StepArgs& a, int kind, int G, int nb)
{
    if constexpr (MULTI) return phase_of_multi(a, kind, G);
    else return phase_of(a, kind, G, nb);
}
template <bool ACT, bool TP, bool GQA, bool BATCH, bool LORA = false, bool MULTI = false>
__global__ void __launch_bounds__(DS_THREADS, 1) decode_step_kernel(const __grid_constant__ StepArgs a)
{
    extern __shared__ __align__(128) unsigned char smem[];
    const int depth = a.depth, nst = 4 * a.depth;
    const int nb = BATCH ? a.bsz : 1;                                                  // sequences of this launch
    unsigned char* ring = smem + ((1024u - (smem_u32(smem) & 1023u)) & 1023u);      // nst x STAGE_STRIDE: pipeline g owns stages [g * depth, (g + 1) * depth)
    // staging slot 0: spt_max K stages; act-order adds slot 1 (H / 128 stages: only the multi-matrix phases, whose K is H, need it --
    // the two matrices a CTA's range can touch have different x_maps)
    // BATCH: nb sequences of a.xst compacted stages each (only the stages the CTA quantises: stage s of a phase sits at (s - s0) mod spt)
    const int xstages = BATCH ? nb * a.xst : a.spt_max + (ACT ? a.H / TILE : 0);
    const uint32_t xs_slot = (uint32_t)a.spt_max * 256u, seg_slot = (uint32_t)a.spt_max * 32u;
    [[maybe_unused]] const uint32_t xs_seq = (uint32_t)a.xst * 256u, seg_seq = (uint32_t)a.xst * 32u;
    unsigned char* xs = ring + (size_t)nst * STAGE_STRIDE;                            // xstages x 16 k8-rows x 16 B: quantised x planes by K stage
    unsigned char* segt = xs + (size_t)xstages * 256;                                  // xstages x 4 x {sum x_q, x scale}
    half* xres = reinterpret_cast<half*>(xs + (MULTI ? stage_area_bytes_multi(xstages, a.n_rep, nb) : stage_area_bytes(xstages, a.n_rep)));    // [nb][H] residual streams (fp16, as the reference keeps them)
    float* parts = reinterpret_cast<float*>(xres + (size_t)nb * a.H);                  // [2 segments][17][PART_LD] attention partials of the warps (+ the new token)
    float* q_s = parts + 2 * 17 * PART_LD;                                             // [2][128] scaled q of the segment's head
    float* kn_s = q_s + 2 * TILE;                                                      // [2][128] newest k row (after rope)
    float* vn_s = kn_s + 2 * TILE;                                                     // [2][128] newest v row
    half* qh_s = reinterpret_cast<half*>(vn_s + 2 * TILE);                             // [2][128] q of the segment's head after rope, fp16 as the reference holds it (unscaled)
    unsigned char* wnorm = reinterpret_cast<unsigned char*>(qh_s + 2 * TILE);          // [H / 8][16 B]: norm weights of the rows this CTA quantises next (by k8-row slot)
    half* xh = reinterpret_cast<half*>(xs);                                            // HEAD: normalised x [nb][H] (xs is free by then)
    float* gparts = reinterpret_cast<float*>(xs);                 // ATT with GQA: [2 segments][n_rep][5][PART_LD] (xs is free then)
    __shared__ __align__(8) unsigned long long full_bar[4 * MAX_DEPTH], empty_bar[4 * MAX_DEPTH];
    __shared__ float s_red[(BATCH ? MAX_BATCH : 1) * DS_NCW];
    __shared__ unsigned long long s_base, s_base_x;
    // The schedule does not depend on the layer (nor, except ATT, on anything but the shapes): this CTA's unit range of every phase,
    // its shares of the buffers it zeroes and the CTA range of every head's attention units are computed ONCE per launch.  (They were
    // 64-bit divisions re-done by every thread in every phase of every layer: 5 % of all instructions executed, in the prologues.)
    __shared__ volatile int s_arrived;                          // phase-end barrier arrivals of this CTA (release fence done)
    __shared__ int s_rng[6][4];                                  // [phase kind]{lo, hi, first K stage lo % spt, K stages to quantise min(hi - lo, spt)}
    __shared__ int s_zr[ZR_COUNT][2];                            // [buffer][lo, hi) in units of 4 floats (ZR_HALF: 2 floats)
    __shared__ unsigned short s_clo[DS_MAX_HEADS], s_chi[DS_MAX_HEADS];        // by virtual head b * heads + h

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int G = (int)gridDim.x, cta = (int)blockIdx.x;

    if (tid == 0) {
        s_arrived = 0;
        for (int i = 0; i < nst; i++) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (tid >= 32 && tid < 38) {
        const Phase p = step_phase<MULTI>(a, tid - 32, G, nb);
        const int lo = range_lo(p.U, cta, p.G), hi = range_lo(p.U, cta + 1, p.G);
        s_rng[tid - 32][0] = lo; s_rng[tid - 32][1] = hi;
        s_rng[tid - 32][2] = (p.spt > 0 && hi > lo) ? lo % p.spt : 0;
        s_rng[tid - 32][3] = p.spt > 0 ? min(hi - lo, p.spt) : 0;
    } else if (tid >= 64 && tid < 64 + ZR_COUNT) {
        const int k = tid - 64;
        int n = k == ZR_QKV ? (a.HQ + 2 * a.HKV) >> 2 : (k == ZR_H ? a.H >> 2 : (k == ZR_GU ? (2 * a.I) >> 2 : (k == ZR_LOGITS ? a.vocab >> 2 : a.H >> 1)));
        if constexpr (BATCH) n *= nb;                              // [nb][width] (ZR_HALF is tensor parallel only)
        s_zr[k][0] = share_lo(n, cta, G); s_zr[k][1] = share_lo(n, cta + 1, G);
    } else if (tid >= 128 && tid < 128 + nb * a.heads) {
        const Phase pa = step_phase<MULTI>(a, PH_ATT, G, nb);
        const int h = tid - 128, kvh = (MULTI ? h % a.heads : h) / a.n_rep;      // a query head's partials come from the CTAs of its KV head (virtual: b * kv_heads + kvh;
                                                                                  // MULTI: virtual query head t * heads + h' of token t reads real KV head h' / n_rep)
        s_clo[h] = (unsigned short)cta_of((long long)kvh * pa.tpm, pa.U, pa.G);
        s_chi[h] = (unsigned short)cta_of((long long)(kvh + 1) * pa.tpm - 1, pa.U, pa.G);
    }
    __syncthreads();

    if (warp >= DS_NCW) {
        // ==================== producer warp of pipeline pq: every 4th stage of the token's HBM stream, in schedule order ====================
        const int pq = warp - DS_NCW;
        int ls = 0; uint32_t par = 0; int issued = 0;                       // ls: stage inside the pipeline's ring; par: parity of the empty completion to wait for
        const uint32_t ring_a = smem_u32(ring) + (uint32_t)pq * depth * STAGE_STRIDE;
        const uint32_t full0 = smem_u32(&full_bar[pq * depth]), empty0 = smem_u32(&empty_bar[pq * depth]);
        int jbase = 0;
        // Stages in flight per pipeline: the cost of a grid-barrier arrival's release fence grows with the bytes the SM has in
        // flight (whole ring in flight: ~4.7 us on an H100; one stage per pipeline: ~1.7 us).  The fences fall while the
        // consumers finish a phase, and the producer is then issuing the first stages of the next phase; so the first `depth`
        // stages of every phase go one at a time (a stage is issued once the pipeline's previous stage has landed), and the
        // rest of the phase, streamed while no barrier is near, keeps up to MID_INFLIGHT stages in flight (DESIGN 3c).
        int nph = 0;                                                          // stages of this pipeline issued in the current phase
        const int kmid = MID_INFLIGHT < depth ? MID_INFLIGHT : depth;
        // The release fence of that arrival waits for every load the SM has in flight, so past the first stage of a phase the
        // producer also waits until its CTA has arrived at the barrier that ends the previous phase (hold_q: phase-end arrivals
        // before this phase).  The fence then finds at most the one stage per pipeline that was issued ahead, usually landed.
        // Tensor parallel plans end O and DOWN with a push instead of a barrier, so they do not hold.
        int hold_q = 0;
        auto acquire = [&](uint32_t tx) -> uint32_t {
            if constexpr (!TP) if (nph == 1 && s_arrived < hold_q) {
                const unsigned long long t0 = gtime();
                while (s_arrived < hold_q) if (gtime() - t0 > WAIT_NS) __trap();
            }
            if (issued >= depth) mbar_wait(empty0 + ls * 8, par ^ 1u);
            const int k = nph < depth ? 1 : kmid;
            if (issued >= k) { int pj = ls - k; uint32_t pp = par; if (pj < 0) { pj += depth; pp ^= 1u; } mbar_wait(full0 + pj * 8, pp); }
            if (lane == 0) mbar_expect_tx(full0 + ls * 8, tx);
            __syncwarp();
            return ring_a + (uint32_t)ls * STAGE_STRIDE;
        };
        auto advance = [&]() { nph++; if (issued < depth) issued++; if (++ls == depth) { ls = 0; par ^= 1u; } };
        // Every byte the ring loads is read once per token: evict-first keeps it from pushing the phase accumulators, attention
        // partials and barrier counter out of L2, which the prologues and barriers read back
        uint64_t pol;
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
        const int ngrow = a.gshift >= 2 ? 1 : (4 >> a.gshift);          // group rows per K stage (groupsize 32: 4, 64: 2, >= 128: 1)
        #pragma unroll 1
        for (int l = 0; l < a.n_layers; l++) {
            const LayerDesc* L = a.layers + l;
            #pragma unroll 1
            for (int ph = PH_QKV; ph <= PH_DOWN; ph++) {
                const Phase p = step_phase<MULTI>(a, ph, G, nb);
                hold_q = l * 5 + ph;
                const int u0 = s_rng[ph][0], u1 = s_rng[ph][1];
                const int i0 = ((pq - jbase) & 3);
                jbase += u1 - u0;
                nph = 0;
                if (ph == PH_ATT) {
                    int h = (u0 + i0) / p.tpm, ch = (u0 + i0) - h * p.tpm;
                    #pragma unroll 1
                    for (int u = u0 + i0; u < u1; u += 4) {
                        const int pos0 = ch * 16;
                        int plen = a.past_len;
                        if constexpr (BATCH && !MULTI) plen = a.past_lens[h / a.kv_heads];        // h: virtual KV head, its rows sit at h * max_seq
                        int nv = plen - pos0; nv = nv < 0 ? 0 : (nv > 16 ? 16 : nv);
                        const uint32_t base = acquire((uint32_t)nv * 512u);
                        if (nv > 0) {
                            // MULTI: h is a real KV head of cache sequence seq; rows [0, past_len) only, never the launch's own
                            const size_t off = ((size_t)(MULTI ? a.seq * a.kv_heads + h : h) * a.max_seq + pos0) * TILE;
                            if (lane == 0) bulk_g2s(base, L->kc + off, (uint32_t)nv * 256u, full0 + ls * 8, pol);
                            if (lane == 1) bulk_g2s(base + 4096, L->vc + off, (uint32_t)nv * 256u, full0 + ls * 8, pol);
                        }
                        advance();
                        ch += 4;
                        while (ch >= p.tpm) { ch -= p.tpm; h++; }
                    }
                    continue;
                }
                if (u0 + i0 >= u1) continue;
                int tile = (u0 + i0) / p.spt, s = (u0 + i0) - tile * p.spt;
                int mi = mat_of_tile(p, tile), ct = tile - mat_tile0(p, mi);
                #pragma unroll 1
                for (int u = u0 + i0; u < u1; u += 4) {
                    const int m = p.mat0 + mi;
                    const uint32_t base = acquire((uint32_t)W_BYTES + (uint32_t)ngrow * 320u);
                    const uint32_t fb = full0 + ls * 8;
                    const int grow = a.gshift >= 2 ? ((s * 4) >> a.gshift) : s * ngrow;
                    if (lane == 0) tma_load_3d(base, &L->tw[m], 0, s * 16, ct * 4, fb, pol);
                    else if (lane == 1) tma_load_2d(base + META_SC, &L->ts[m], ct * TILE, grow, fb, pol);
                    else if (lane == 2) tma_load_2d(base + META_ZQ, &L->tz[m], ct * 16, grow, fb, pol);
                    advance();
                    s += 4;
                    while (s >= p.spt) { s -= p.spt; if (++ct == mat_tiles(p, mi)) { ct = 0; mi++; } }
                }
            }
        }
        {
            const int u0 = s_rng[PH_HEAD][0], u1 = s_rng[PH_HEAD][1];
            const int i0 = ((pq - jbase) & 3);
            nph = 0;
            hold_q = a.n_layers * 5;
            const long long total = (long long)a.vocab * a.H * 2;
            const unsigned char* src = reinterpret_cast<const unsigned char*>(a.lm_head);
            #pragma unroll 1
            for (int u = u0 + i0; u < u1; u += 4) {
                const long long off = (long long)u * W_BYTES;
                const uint32_t bytes = (uint32_t)((total - off) < W_BYTES ? (total - off) : W_BYTES);
                const uint32_t base = acquire(bytes);
                if (lane == 0) bulk_g2s(base, src + off, bytes, full0 + ls * 8, pol);
                advance();
            }
        }
        return;
    }

    // ======================================================= consumer warps =======================================================
    const int wn = warp & 3, wk = warp >> 2;             // wk: pipeline; wn: 32-column quarter of the tile (ATT: 4 positions, HEAD: 2 chunks)
    const int g = lane >> 2, t = lane & 3;
    const int pg = (g >> 1) | ((g & 1) << 2);            // column chunk of this lane (bank-conflict-free against the 128B swizzle)
    const int lane_col = wn * 32 + 4 * pg;
    const uint32_t ring_a = smem_u32(ring) + (uint32_t)wk * depth * STAGE_STRIDE;
    const uint32_t full0 = smem_u32(&full_bar[wk * depth]), empty0 = smem_u32(&empty_bar[wk * depth]);
    int ls = 0; uint32_t par = 0;                        // this pipeline's ring position (every warp of the pipeline visits every stage)
    auto stamp = [&](int l, int ev) { if (a.trace && tid == 0 && l < TRACE_LAYERS) a.trace[((size_t)cta * TRACE_LAYERS + l) * 24 + ev] = gtime(); };
    int jbase = 0;                                       // stages this CTA has been through (same count as the producers)
    if (tid == 0) {
        unsigned long long v;
        asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(a.bar) : "memory");
        s_base = v - v % (unsigned long long)G;          // at most G - 1 CTAs of THIS launch can have arrived already
        s_base_x = TP ? (unsigned long long)__ldcg(a.launch_ctr) : 0ull;
    }
    consumer_sync();
    unsigned long long target = s_base + (unsigned long long)G;
    const unsigned epoch0 = (unsigned)s_base_x * (unsigned)(2 * a.n_layers) + 1u;      // epoch of (layer l, o / down) = epoch0 + 2 l + {0, 1}

    auto zero_share = [&](float* buf, int which) {        // this CTA's share of a float buffer (its length % 4 == 0)
        const int lo = s_zr[which][0], hi = s_zr[which][1];
        for (int i = lo + tid; i < hi; i += DS_CONSUMERS) reinterpret_cast<float4*>(buf)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    };

    // ---- launch start: all accumulators and the logits to zero (robust against an aborted previous launch), then barrier ----
    zero_share(a.acc_qkv, ZR_QKV); zero_share(a.acc_o, ZR_H); zero_share(a.acc_gu, ZR_GU); zero_share(a.acc_d, ZR_H);
    if (a.logits) zero_share(a.logits, ZR_LOGITS);
    if constexpr (LORA)
        for (int i = share_lo(a.lora_t4, cta, G) + tid; i < share_lo(a.lora_t4, cta + 1, G); i += DS_CONSUMERS)
            reinterpret_cast<float4*>(a.lora_t)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = tid; i < nb * a.H / 8; i += DS_CONSUMERS)
        reinterpret_cast<uint4*>(xres)[i] = __ldg(reinterpret_cast<const uint4*>(a.x_in) + i);

    const int rpg = a.gshift >= 2 ? 16 : (4 << a.gshift);          // k8-rows per quantisation segment (a segment never spans stages)

    // Norm weights of the rows this CTA will quantise in the NEXT norm phase are constants: they are copied into shared memory
    // with cp.async BEFORE the grid barrier (no registers held), so the phase prologue is left with one L2 round trip (the
    // accumulator) instead of two.  Slot r of wnorm holds the weights of row r of the staging order.
    auto preload_norm = [&](const half* nw, const Phase& p) {
        if constexpr (ACT) return;                          // act-order: the getter gathers the weights itself
        const int n = s_rng[p.kind][3], s0 = s_rng[p.kind][2];
        for (int r = tid; r < n * 16; r += DS_CONSUMERS) {
            int s = s0 + (r >> 4); if (s >= p.spt) s -= p.spt;
            asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" :: "r"(smem_u32(wnorm) + (uint32_t)r * 16u), "l"(nw + (size_t)(s * 16 + (r & 15)) * 8) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    preload_norm(a.layers[0].ln1, phase_of(a, PH_QKV, G, nb));
    grid_barrier(a.bar, target, (unsigned)G, tid);
    if (TP && cta == 0 && tid == 0) *a.launch_ctr = (unsigned)s_base_x + 1u;      // every CTA has read it (it is past the barrier)

    // ---- per sequence b (residual stream b, accumulator row b, s_red row b): residual add (fp16(x + fp32 delta), the rounding point of
    // q4_matmul's no_zero epilogue) + row factor of the RMS norm into rmb[b].  Without BATCH nb is the constant 1 and the loops fold away.
    float rmb[MAX_BATCH] = {0.f, 0.f, 0.f, 0.f};
    auto residual_and_norm = [&](const float* delta, const uint2* slots = nullptr, unsigned epoch = 0u) {
        asm volatile("cp.async.wait_all;" ::: "memory");
        for (int b = 0; b < nb; b++) {
            float ss = 0.f;
            uint4* xr = reinterpret_cast<uint4*>(xres + (size_t)b * a.H);
            for (int i = tid; i < a.H / 8; i += DS_CONSUMERS) {
                uint4 xv = xr[i];
                half2* h = reinterpret_cast<half2*>(&xv);
                if (delta) {
                    const float* dp = delta + (size_t)b * a.H + i * 8;
                    const float4 own0 = ldcg4(dp), own1 = ldcg4(dp + 4);
                    float4 d0 = own0, d1 = own1;
                    if constexpr (TP) if (slots) {
                        // tensor parallel (nb is 1): the sum over ALL ranks' partials in rank order (bitwise identical on every rank); the
                        // peers' partials sit in this rank's slots as {value, epoch} pairs, polled until the epoch of this (layer, phase) shows up
                        d0 = make_float4(0.f, 0.f, 0.f, 0.f); d1 = d0;
                        for (int r = 0; r < a.tp_world; r++) {
                            float e[8];
                            if (r == a.tp_rank) {
                                e[0] = own0.x; e[1] = own0.y; e[2] = own0.z; e[3] = own0.w; e[4] = own1.x; e[5] = own1.y; e[6] = own1.z; e[7] = own1.w;
                            } else {
                                const uint4* sp = reinterpret_cast<const uint4*>(slots + (size_t)r * a.H + i * 8);
                                #pragma unroll
                                for (int q = 0; q < 4; q++) {
                                    uint4 v;
                                    asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(sp + q) : "memory");
                                    if (v.y != epoch || v.w != epoch) {
                                        const unsigned long long t0 = gtime();
                                        unsigned spin = 0;
                                        do {
                                            asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(sp + q) : "memory");
                                            if ((++spin & 1023u) == 0 && gtime() - t0 > WAIT_NS) __trap();
                                        } while (v.y != epoch || v.w != epoch);
                                    }
                                    e[2 * q] = __uint_as_float(v.x); e[2 * q + 1] = __uint_as_float(v.z);
                                }
                            }
                            d0.x += e[0]; d0.y += e[1]; d0.z += e[2]; d0.w += e[3]; d1.x += e[4]; d1.y += e[5]; d1.z += e[6]; d1.w += e[7];
                        }
                    }
                    float2 f;
                    f = __half22float2(h[0]); h[0] = __floats2half2_rn(f.x + d0.x, f.y + d0.y);
                    f = __half22float2(h[1]); h[1] = __floats2half2_rn(f.x + d0.z, f.y + d0.w);
                    f = __half22float2(h[2]); h[2] = __floats2half2_rn(f.x + d1.x, f.y + d1.y);
                    f = __half22float2(h[3]); h[3] = __floats2half2_rn(f.x + d1.z, f.y + d1.w);
                    xr[i] = xv;
                }
                #pragma unroll
                for (int j = 0; j < 4; j++) { const float2 f = __half22float2(h[j]); ss = fmaf(f.x, f.x, ss); ss = fmaf(f.y, f.y, ss); }
            }
            #pragma unroll
            for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
            if (lane == 0) s_red[b * DS_NCW + warp] = ss;
        }
        consumer_sync();                                      // also publishes the updated xres
        #pragma unroll
        for (int b = 0; b < MAX_BATCH; b++) {
            if (b >= nb) break;
            float tot = 0.f;
            #pragma unroll
            for (int w = 0; w < DS_NCW; w++) tot += s_red[b * DS_NCW + w];      // same order in every thread
            rmb[b] = __half2float(__float2half_rn(rsqrtf(tot / (float)a.H + a.eps)));      // rms_norm.cu:113-116
        }
    };
    // a select chain, not rmb[b]: a run-time index would put rmb in local memory.  Without BATCH b is always 0, which the compiler
    // cannot see where b is computed (lora_a's i >> 4)
    auto rm_of = [&](int b) { return (!BATCH || b == 0) ? rmb[0] : b == 1 ? rmb[1] : b == 2 ? rmb[2] : rmb[3]; };

    // ---- quantise the K stages [s0, s0 + n) (cyclic mod spt) of the phase input into xs / segt; `get(k8, it)` yields 8 fp16 values ----
    // BATCH: slot is the sequence, and stage s0 + j goes to compacted stage j of that sequence's area
    // RPGC = k8-rows per quantisation segment at compile time (16: groupsize >= 128, the common case: unrolled shuffles, shifts instead
    // of divisions) or 0 = the run-time value rpg (groupsize 32 / 64)
    auto stage_x = [&](auto rpg_c, int s0, int n, int spt, auto get, int slot) {
        constexpr int RPGC = decltype(rpg_c)::value;
        const int rp = RPGC ? RPGC : rpg;
        unsigned char* xs_w = xs; unsigned char* seg_w = segt;
        if constexpr (ACT) { xs_w += (size_t)slot * xs_slot; seg_w += (size_t)slot * seg_slot; }
        if constexpr (BATCH) { xs_w += (size_t)slot * xs_seq; seg_w += (size_t)slot * seg_seq; }
        const int nrows = n * 16;
        int it = 0;
        for (int base = 0; base < nrows; base += DS_CONSUMERS, it++) {
            const int r = base + tid;
            const bool act = r < nrows;
            int s = s0 + (r >> 4); if (s >= spt) s -= spt;
            const int rr = r & 15;
            const uint4 hv = act ? get(s * 16 + rr, it) : make_uint4(0, 0, 0, 0);
            float mx = row_absmax(hv);
            if constexpr (RPGC != 0) {
                #pragma unroll
                for (int o = RPGC >> 1; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            } else {
                for (int o = rp >> 1; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            }
            uint4 q;
            int sum = quantise_row(hv, mx > 0.f ? 32639.0f / mx : 0.f, q);
            if constexpr (RPGC != 0) {
                #pragma unroll
                for (int o = RPGC >> 1; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
            } else {
                for (int o = rp >> 1; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
            }
            if (act) {
                const int sx = BATCH ? (r >> 4) : s;
                *reinterpret_cast<uint4*>(xs_w + (size_t)sx * 256 + rr * 16) = q;
                if ((rr & (rp - 1)) == 0)
                    *reinterpret_cast<float2*>(seg_w + (size_t)sx * 32 + (rr / rp) * 8) = make_float2(__int_as_float(sum), mx * (1.0f / 32639.0f));
            }
        }
    };
    auto stage_xd = [&](int s0, int n, int spt, auto get, int slot = 0) {
        if (rpg == 16) stage_x(std::integral_constant<int, 16>{}, s0, n, spt, get, slot);
        else stage_x(std::integral_constant<int, 0>{}, s0, n, spt, get, slot);
    };
    // sequence b's residual stream, normalised with its row factor rm and the norm weights preload_norm put in wnorm
    auto norm_get = [&](int b, float rm) {
        const uint4* xr = reinterpret_cast<const uint4*>(xres + (size_t)b * a.H);
        return [=](int k8, int it) -> uint4 {
            uint4 xv = xr[k8];
            const uint4 wv = reinterpret_cast<const uint4*>(wnorm)[it * DS_CONSUMERS + tid];
            const half2 rm2 = __float2half2_rn(rm);
            half2* h = reinterpret_cast<half2*>(&xv); const half2* w2 = reinterpret_cast<const half2*>(&wv);
            #pragma unroll
            for (int i = 0; i < 4; i++) h[i] = __hmul2(__hmul2(h[i], rm2), w2[i]);      // rms_norm.cu:118-131
            return xv;
        };
    };

    // ---- stage the phase input for every matrix the CTA's unit range touches.  Without act-order all matrices of a phase share x
    // (one staging); with act-order each matrix gathers x through its own x_map (q4_matmul.cu:239-299 / column_remap.cu:27-34), so a
    // range that crosses a matrix boundary stages twice, into slot (matrix - first matrix).  make_get(m) returns the 8-value getter.
    auto stage_phase = [&](const Phase& p, int u0, int u1, auto make_get) {
        if (u1 <= u0) return;
        const int mi0 = mat_of_tile(p, u0 / p.spt), mi1 = ACT ? mat_of_tile(p, (u1 - 1) / p.spt) : mi0;
        for (int mi = mi0; mi <= mi1; mi++) {
            const int m_lo = mat_tile0(p, mi) * p.spt, m_hi = m_lo + mat_tiles(p, mi) * p.spt;
            const int ua = ACT ? max(u0, m_lo) : u0, ub = ACT ? min(u1, m_hi) : u1;
            stage_xd(ua % p.spt, min(ub - ua, p.spt), p.spt, make_get(p.mat0 + mi), mi - mi0);
        }
    };
    // x (residual stream in shared memory) -> (x * rm) * w, gathered through an x_map when there is one (rms_norm.cu:118-131)
    auto norm_get_map = [&](const half* nw, float rmf, const uint32_t* map) {
        return [=](int k8, int) -> uint4 {
            uint32_t idx[8];
            load_map8(map, k8, idx);
            const half2 rm2 = __float2half2_rn(rmf);
            uint4 r; half2* h = reinterpret_cast<half2*>(&r);
            #pragma unroll
            for (int i = 0; i < 4; i++) {
                const half2 xv = __halves2half2(xres[idx[2 * i]], xres[idx[2 * i + 1]]);
                const half2 wv = __halves2half2(__ldg(nw + idx[2 * i]), __ldg(nw + idx[2 * i + 1]));
                h[i] = __hmul2(__hmul2(xv, rm2), wv);
            }
            return r;
        };
    };

    // ---- GEMV phase body: this pipeline's stages of the CTA's unit range, this warp's 32 columns ----
    // UPSEG = units (of 4 k8-rows = 32 k) per quantisation segment, compile-time: 4 (groupsize >= 128), 2 (64), 1 (32).
    auto gemv_t = [&](auto upseg_c, const Phase& p, int u0, int u1) {
        constexpr int UPSEG = decltype(upseg_c)::value;
        int u = u0 + ((wk - jbase) & 3);                // stage j of the CTA goes to pipeline j & 3
        if (u >= u1) return;
        int tile = u / p.spt, s = u - tile * p.spt;
        int cur_tile = tile;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        [[maybe_unused]] const size_t acc_ld = (size_t)(p.tq + (p.nmat - 1) * p.tpm) * TILE;      // BATCH: accumulator row of a sequence
        auto flush_tile = [&]() {
            if constexpr (BATCH) { if (t < nb) red_add_v4(p.acc + t * acc_ld + (size_t)cur_tile * TILE + lane_col, acc[0], acc[1], acc[2], acc[3]); }
            else if (t == 0) red_add_v4(p.acc + (size_t)cur_tile * TILE + lane_col, acc[0], acc[1], acc[2], acc[3]);     // tiles are numbered matrix by matrix
            acc[0] = acc[1] = acc[2] = acc[3] = 0.f;
        };
        // every address below is a 32-bit shared-memory address built from per-lane constants computed once per phase
        // B column n of the MMA is supplied by the lanes with g == n: 0 = high-byte plane of x, 1 = low-byte plane.  Columns 2..7 only
        // feed D columns 2..7, which live in lanes t >= 1 and are never read -- so those lanes may load anything (they load plane g & 1).
        // BATCH: columns 2b, 2b + 1 carry sequence b (idle columns repeat the last sequence), so lane t's D columns 2t, 2t + 1 are
        // sequence t's result: every lane uses the segment sums of its own sequence t and lanes t < nb flush.
        uint32_t x_lane = smem_u32(xs) + t * 16 + (g & 1) * 8;
        if constexpr (BATCH) x_lane += (uint32_t)min(g >> 1, nb - 1) * xs_seq;
        constexpr uint32_t xstage = 256u, xunit = 64u;
        const uint32_t w_lane = (uint32_t)(wn * BOX_BYTES + t * 128 + ((pg ^ t) << 4));              // k8-rows t, t + 8 (r & 7 == t)
        const uint32_t w_lane4 = w_lane + 512u + ((pg & 4) ? -64 : 64);                              // k8-rows t + 4, t + 12: chunk (pg ^ t) ^ 4
        const uint32_t sc_lane = (uint32_t)(META_SC + lane_col * 2), zq_lane = (uint32_t)(META_ZQ + (lane_col >> 3) * 4);
        const uint32_t zshift = (uint32_t)((lane_col & 4) * 4);
        uint32_t seg_a = smem_u32(segt);
        if constexpr (BATCH) seg_a += (uint32_t)min(t, nb - 1) * seg_seq;
        [[maybe_unused]] const int s0c = s_rng[p.kind][2];                                  // BATCH: first staged K stage (compacted index 0)
        // NOTE: everything act-order specific is under `if constexpr`: with plain runtime-constant code in its place ptxas produced a
        // 10 % slower plain kernel (measured by A/B builds on one box: any one of these blocks removed restored the speed)
        [[maybe_unused]] int mi_first = 0;                  // staging slot of a tile = its matrix - the first matrix of the CTA's range
        [[maybe_unused]] uint32_t xoff = 0u, soff = 0u;
        if constexpr (ACT) { mi_first = mat_of_tile(p, u0 / p.spt); xoff = (uint32_t)(mat_of_tile(p, cur_tile) - mi_first) * xs_slot; soff = (uint32_t)(mat_of_tile(p, cur_tile) - mi_first) * seg_slot; }
        bool ready = mbar_try(full0 + ls * 8, par);
        for (; u < u1; u += 4) {
            if (tile != cur_tile) {
                flush_tile(); cur_tile = tile;
                if constexpr (ACT) { const uint32_t sl = (uint32_t)(mat_of_tile(p, tile) - mi_first); xoff = sl * xs_slot; soff = sl * seg_slot; }
            }
            const uint32_t tok = mbar_wait_tok(full0 + ls * 8, par, ready);
            const int ls_cur = ls;
            if (++ls == depth) { ls = 0; par ^= 1u; }
            // probe the NEXT stage's barrier now: its ~90-cycle answer overlaps this stage's work
            ready = (u + 4 < u1) ? mbar_try(full0 + ls * 8, par) : false;
            float dep = 0.f;
            if (!(a.debug & 1)) {
                const uint32_t sb = ring_a + (uint32_t)ls_cur * STAGE_STRIDE + tok;
                int sx = s;
                if constexpr (BATCH) { sx = s - s0c; if (sx < 0) sx += p.spt; }
                uint32_t xr = x_lane + (uint32_t)sx * xstage + tok;
                if constexpr (ACT) xr += xoff;
                uint4 w[4]; uint2 xv[4];
                w[0] = lds128(sb + w_lane);         w[1] = lds128(sb + w_lane4);
                w[2] = lds128(sb + w_lane + 1024);  w[3] = lds128(sb + w_lane4 + 1024);
                #pragma unroll
                for (int q = 0; q < 4; q++) xv[q] = lds64(xr + q * xunit);
                // per-segment parameters (all independent of the MMAs: issued up front)
                constexpr int NSEG = 4 / UPSEG;
                uint2 sc2[NSEG]; uint32_t zw[NSEG]; uint2 sg[NSEG];
                #pragma unroll
                for (int e = 0; e < NSEG; e++) {
                    const int row = UPSEG == 4 ? 0 : e;
                    sc2[e] = lds64(sb + sc_lane + row * 256);
                    zw[e] = lds32(sb + zq_lane + row * 64);
                    if constexpr (ACT) sg[e] = lds64(seg_a + (uint32_t)s * 32u + e * 8 + soff + tok);
                    else sg[e] = lds64(seg_a + (uint32_t)sx * 32u + e * 8 + tok);
                }
                // two independent accumulator sets (even / odd units) halve the dependent IMMA chain
                int ia[2][8];
                #pragma unroll
                for (int q = 0; q < 4; q++) {
                    const uint32_t M4 = 0x0f0f0f0fu;
                    const uint32_t lo0 = w[q].x & M4, hi0 = (w[q].x >> 4) & M4, lo1 = w[q].y & M4, hi1 = (w[q].y >> 4) & M4;
                    const uint32_t lo2 = w[q].z & M4, hi2 = (w[q].z >> 4) & M4, lo3 = w[q].w & M4, hi3 = (w[q].w >> 4) & M4;
                    const int set = UPSEG == 1 ? 0 : (q & 1);
                    int (&aA)[4] = *reinterpret_cast<int (*)[4]>(&ia[set][0]);
                    int (&aB)[4] = *reinterpret_cast<int (*)[4]>(&ia[set][4]);
                    const bool first = UPSEG == 1 || (q % UPSEG) < 2;        // first unit of this set in the segment
                    if (first) {
                        imma_z(aA, lo0, lo1, hi0, hi1, xv[q].x, xv[q].y);
                        imma_z(aB, lo2, lo3, hi2, hi3, xv[q].x, xv[q].y);
                    } else {
                        imma(aA, lo0, lo1, hi0, hi1, xv[q].x, xv[q].y);
                        imma(aB, lo2, lo3, hi2, hi3, xv[q].x, xv[q].y);
                    }
                    if ((q + 1) % UPSEG == 0) {
                        // segment complete: acc += scale * sx * (256 * sum a q + sum b q - zp * sum x_q)
                        const int e = q / UPSEG;
                        const int sxq = (int)sg[e].x; const float sx = __uint_as_float(sg[e].y);
                        const half2 s01 = *reinterpret_cast<const half2*>(&sc2[e].x), s23 = *reinterpret_cast<const half2*>(&sc2[e].y);
                        const float cs4[4] = {__low2float(s01), __high2float(s01), __low2float(s23), __high2float(s23)};
                        const uint32_t z4 = zw[e] >> zshift;
                        #pragma unroll
                        for (int c = 0; c < 4; c++) {
                            // lane t == 0: D(row g / g+8, col 0 = plane a, col 1 = plane b); column c of this lane = MMA (c >> 1), row half (c & 1)
                            const int jj = (c >> 1) * 4 + (c & 1) * 2;
                            const int zp = (int)((z4 >> (4 * c)) & 0xfu) + 1;
                            int va = ia[0][jj], vb = ia[0][jj + 1];
                            if (UPSEG > 1) { va += ia[1][jj]; vb += ia[1][jj + 1]; }
                            const int val = va * 256 + vb - zp * sxq;
                            acc[c] = fmaf(cs4[c] * sx, (float)val, acc[c]);
                        }
                    }
                }
                dep = acc[0] + acc[1] + acc[2] + acc[3];
            }
            __syncwarp();
            if (lane == 0) mbar_arrive_dep(empty0 + ls_cur * 8, dep);
            s += 4; while (s >= p.spt) { s -= p.spt; tile++; }
        }
        flush_tile();
    };
    auto gemv = [&](const Phase& p, int u0, int u1) {
        if (rpg == 16) gemv_t(std::integral_constant<int, 4>{}, p, u0, u1);
        else if (rpg == 8) gemv_t(std::integral_constant<int, 2>{}, p, u0, u1);
        else gemv_t(std::integral_constant<int, 1>{}, p, u0, u1);
    };

    // ---- LoRA (LORA kernels only).  LA step of an adapted phase: t[b][j] += x_b[k] * A[k, j] over this CTA's (matrix, K stage) units
    // (decode_step_sched.h), x_b being sequence b's phase input in the checkpoint's input order -- never gathered through an x_map: the
    // rows of A are in that order -- as make_get(b)(k8) yields it, 8 fp16 values at a time.  fp32 products and sums, fp32 red.add into
    // t in L2.  Returns whether the phase is adapted: the caller then runs a grid barrier, after which t is complete.
    auto lora_a = [&](int l, const Phase& p, auto make_get) -> bool {
        const LoraMat* lm = a.lora + l * 7 + p.mat0;
        int js[3] = {0, 0, 0}, na = 0;
        for (int m = 0; m < p.nmat; m++) if (lm[m].rank > 0) js[na++] = m;
        if (na == 0) return false;
        float* lx = parts;                                   // [nb][128] x of the unit's K stage (the attention partials are free here)
        float* lt = parts + MAX_BATCH * TILE;                // [nb][rank] this unit's share of t
        const int U = lora_units(na, p.spt);
        for (int v = share_lo(U, cta, G); v < share_lo(U, cta + 1, G); v++) {
            const int s = v % p.spt;
            const LoraMat m = lm[js[v / p.spt]];
            for (int i = tid; i < nb * 16; i += DS_CONSUMERS) {
                const int b = i >> 4, r = i & 15;
                const uint4 hv = make_get(b)(s * 16 + r);
                const half2* h = reinterpret_cast<const half2*>(&hv);
                #pragma unroll
                for (int q = 0; q < 4; q++) { const float2 f = __half22float2(h[q]); lx[b * TILE + r * 8 + 2 * q] = f.x; lx[b * TILE + r * 8 + 2 * q + 1] = f.y; }
            }
            for (int i = tid; i < nb * m.rank; i += DS_CONSUMERS) lt[i] = 0.f;
            consumer_sync();
            const int nkg = DS_CONSUMERS / m.rank;           // k groups: thread (kg, j) takes rows kg, kg + nkg, ... of column j
            if (tid < nkg * m.rank) {
                const int j = tid % m.rank, kg = tid / m.rank;
                const half* ap = m.a + (size_t)s * TILE * m.rank + j;
                float acc[MAX_BATCH] = {0.f, 0.f, 0.f, 0.f};
                for (int k = kg; k < TILE; k += nkg) {
                    const float w = __half2float(__ldg(ap + (size_t)k * m.rank));
                    #pragma unroll
                    for (int b = 0; b < MAX_BATCH; b++) if (b < nb) acc[b] = fmaf(lx[b * TILE + k], w, acc[b]);
                }
                #pragma unroll
                for (int b = 0; b < MAX_BATCH; b++) if (b < nb) atomicAdd(lt + b * m.rank + j, acc[b]);
            }
            consumer_sync();
            for (int i = tid; i < nb * m.rank; i += DS_CONSUMERS) atomicAdd(a.lora_t + m.t_off + i, lt[i]);     // t: [b][rank]
            consumer_sync();                                  // lx / lt are reused by the next unit
        }
        return true;
    };
    // B term, after the GEMV of the phase: every tile of an adapted matrix whose K stage 0 this CTA owns gets
    // acc[b][tile columns] += sum_j fp16(t[b][j]) * B[j, columns], in fp32 (t rounded to fp16 where the reference rounds lora_temp)
    auto lora_b = [&](int l, const Phase& p, int u0, int u1) {
        if (u1 <= u0) return;
        const LoraMat* lm = a.lora + l * 7 + p.mat0;
        const size_t acc_ld = (size_t)(p.tq + (p.nmat - 1) * p.tpm) * TILE;      // accumulator row of a sequence
        const int c = tid & (TILE - 1), jq = tid >> 7;                          // column of the tile, quarter of the rank
        for (int tile = lora_b_first(p, u0); tile * p.spt < u1; tile++) {
            const int mi = mat_of_tile(p, tile);
            const LoraMat m = lm[mi];
            if (m.rank == 0) continue;
            const int n = mat_tiles(p, mi) * TILE;
            const half* bp = m.b + (size_t)(tile - mat_tile0(p, mi)) * TILE + c;
            for (int b = 0; b < nb; b++) {
                const float* tp = a.lora_t + m.t_off + b * m.rank;
                float sum = 0.f;
                for (int j = jq; j < m.rank; j += DS_CONSUMERS / TILE)
                    sum = fmaf(__half2float(__float2half_rn(__ldcg(tp + j))), __half2float(__ldg(bp + (size_t)j * n)), sum);
                atomicAdd(p.acc + b * acc_ld + (size_t)tile * TILE + c, sum);
            }
        }
    };
    // LA inputs: sequence b's residual stream normalised with its row factor and the norm weights nw (as norm_get, un-gathered)
    auto lora_norm_get = [&](const half* nw, int b, float rmf) {
        const uint4* xr = reinterpret_cast<const uint4*>(xres + (size_t)b * a.H);
        return [=](int k8) -> uint4 {
            uint4 xv = xr[k8];
            const uint4 wv = __ldg(reinterpret_cast<const uint4*>(nw) + k8);
            const half2 rm2 = __float2half2_rn(rmf);
            half2* h = reinterpret_cast<half2*>(&xv); const half2* w2 = reinterpret_cast<const half2*>(&wv);
            #pragma unroll
            for (int i = 0; i < 4; i++) h[i] = __hmul2(__hmul2(h[i], rm2), w2[i]);
            return xv;
        };
    };

    // tensor parallel: after the local barrier, this CTA's share of the rank's reduced partial goes into every peer's slot [tp_rank]
    // as {value, epoch} pairs (8-byte stores; two pairs per 16-byte store are fine: each pair is validated on its own)
    auto push_partial = [&](const float* acc, uint2* const* push, unsigned epoch, int l, int ev) {
        grid_barrier(a.bar, target, (unsigned)G, tid);                     // the rank's partial is complete in L2
        stamp(l, ev);
        const int lo = s_zr[ZR_HALF][0], n2 = s_zr[ZR_HALF][1] - lo;                               // in units of 2 floats
        for (int i = tid; i < n2 * (a.tp_world - 1); i += DS_CONSUMERS) {
            int r = i / n2; const int j = i - r * n2;
            if (r >= a.tp_rank) r++;
            const float2 v = __ldcg(reinterpret_cast<const float2*>(acc) + lo + j);
            uint4 o = make_uint4(__float_as_uint(v.x), epoch, __float_as_uint(v.y), epoch);
            asm volatile("st.relaxed.sys.global.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(reinterpret_cast<uint4*>(push[r]) + lo + j), "r"(o.x), "r"(o.y), "r"(o.z), "r"(o.w) : "memory");
        }
        stamp(l, ev + 1);
        if (a.tp_reduce) {
            // total this CTA's share over the ranks in rank order (peers' pairs polled until the epoch shows up), write it back into the
            // accumulator, and publish with a second local barrier: the prologue that follows reads ONE complete vector
            const uint4* rx = reinterpret_cast<const uint4*>(push == a.push_o ? a.slots_o : a.slots_d);
            for (int j = tid; j < n2; j += DS_CONSUMERS) {
                const float2 own = __ldcg(reinterpret_cast<const float2*>(acc) + lo + j);
                float2 tot = make_float2(0.f, 0.f);
                for (int r = 0; r < a.tp_world; r++) {
                    float2 e = own;
                    if (r != a.tp_rank) {
                        const uint4* sp = rx + (size_t)r * (a.H >> 1) + lo + j;
                        uint4 v;
                        const unsigned long long t0 = gtime();
                        unsigned spin = 0;
                        do {
                            asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(sp) : "memory");
                            if ((++spin & 1023u) == 0 && gtime() - t0 > WAIT_NS) __trap();
                        } while (v.y != epoch || v.w != epoch);
                        e = make_float2(__uint_as_float(v.x), __uint_as_float(v.z));
                    }
                    tot.x += e.x; tot.y += e.y;
                }
                reinterpret_cast<float2*>(const_cast<float*>(acc))[lo + j] = tot;
            }
            grid_barrier(a.bar, target, (unsigned)G, tid);
        }
    };

    // ---- ATT under grouped-query attention (n_rep > 1).  A unit is (KV head, 16-position chunk) and its stage of K/V serves all n_rep
    // query heads of the group: warp wn of a pipeline takes the query heads r = wn, wn + 4, ... over all 16 positions of the stage.  The
    // running (m, l, o) of a (segment, query head, pipeline) lives in shared memory (gparts, on the x staging area, which is dead between
    // the QKV GEMV and the O prologue), so a query head of a segment ends with 4 pipeline partials + the new token's, combined into the
    // CTA's slot of att_part as in the multi-head path.
    auto att_gqa = [&](const LayerDesc* L, int u0, int u1, int nph, int h0, int nseg) {
        const int nr = MULTI ? a.n_rep * nb : a.n_rep;                  // query vectors per KV head (MULTI: token t, query head r at t * n_rep + r)
        const int nt = MULTI ? nb : 1;                                  // new k / v rows per KV head
        const float scale = rsqrtf((float)TILE);
        const int l16 = lane & 15, sub = lane >> 4;
        half* gq = reinterpret_cast<half*>(xs + gqa_qh_off(nr));        // [2][nr][128] q after rope, fp16 (unscaled)
        float* gkn = reinterpret_cast<float*>(xs + gqa_kn_off(nr));    // [2][nt][128] newest k rows (after rope)
        float* gvn = gkn + 2 * nt * TILE;                               // [2][nt][128] newest v rows
        auto owner = [&](int kvh) { return min(u1, (kvh + 1) * nph) == (kvh + 1) * nph; };      // holds the KV head's last chunk
        // BATCH: kvh is a virtual KV head b * kv_heads + kvh' -- its sequence's context, rope row and accumulator row.  MULTI: kvh is
        // a real KV head and every token attends the same history
        auto plen_of = [&](int kvh) { if constexpr (BATCH && !MULTI) return a.past_lens[kvh / a.kv_heads]; else return a.past_len; };
        const size_t qkv_ld = (size_t)a.HQ + 2 * a.HKV;
        const half* sr1 = a.sin + (size_t)a.past_len * TILE;
        const half* cr1 = a.cos + (size_t)a.past_len * TILE;
        // rope q of every query head of the segments (rope.cu:48-67, as the multi-head path); rope k and write the k / v cache rows
        // once per KV head, by its owner; every pipeline partial to neutral
        if constexpr (MULTI) {
            // token t at position past_len + t: its q from accumulator row t, its k / v rows into row past_len + t of sequence seq
            for (int i = tid; i < nseg * nr * TILE; i += DS_CONSUMERS) {
                const int d = i & 127, w = i >> 7, sg = w / nr, j = w - sg * nr, t = j / a.n_rep;
                const int qh = (h0 + sg) * a.n_rep + (j - t * a.n_rep);
                const half* sr = a.sin + (size_t)(a.past_len + t) * TILE;
                const half* cr = a.cos + (size_t)(a.past_len + t) * TILE;
                const float* aq = a.acc_qkv + t * qkv_ld + (size_t)qh * TILE;
                const half qv = __float2half_rn(__ldcg(aq + d)), qo = __float2half_rn(__ldcg(aq + (d ^ 64)));
                const half sn = d < 64 ? __hneg(sr[d]) : sr[d];
                gq[w * TILE + d] = __hfma(qv, cr[d], __hmul(qo, sn));
            }
            for (int i = tid; i < nseg * nt * TILE; i += DS_CONSUMERS) {
                const int d = i & 127, w = i >> 7, sg = w / nt, t = w - sg * nt, kvh = h0 + sg;
                if (!owner(kvh)) continue;
                const int pos = a.past_len + t;
                const half* sr = a.sin + (size_t)pos * TILE;
                const half* cr = a.cos + (size_t)pos * TILE;
                const half sn = d < 64 ? __hneg(sr[d]) : sr[d];
                const float* ak = a.acc_qkv + t * qkv_ld + a.HQ + (size_t)kvh * TILE;
                const half kv = __float2half_rn(__ldcg(ak + d)), ko = __float2half_rn(__ldcg(ak + (d ^ 64)));
                const half kr = __hfma(kv, cr[d], __hmul(ko, sn));
                const half vv = __float2half_rn(__ldcg(ak + a.HKV + d));
                gkn[w * TILE + d] = __half2float(kr); gvn[w * TILE + d] = __half2float(vv);
                const size_t off = (((size_t)a.seq * a.kv_heads + kvh) * a.max_seq + pos) * TILE + d;
                L->kc[off] = kr; L->vc[off] = vv;
            }
        } else {
        for (int i = tid; i < nseg * nr * TILE; i += DS_CONSUMERS) {
            const int d = i & 127, w = i >> 7, sg = w / nr;
            int qh = (h0 + sg) * nr + (w - sg * nr);
            const half* sr = BATCH ? a.sin + (size_t)plen_of(h0 + sg) * TILE : sr1;
            const half* cr = BATCH ? a.cos + (size_t)plen_of(h0 + sg) * TILE : cr1;
            const float* aq = a.acc_qkv;
            if constexpr (BATCH) { const int b = (h0 + sg) / a.kv_heads; aq += b * qkv_ld; qh -= b * a.heads; }
            aq += (size_t)qh * TILE;
            const half qv = __float2half_rn(__ldcg(aq + d)), qo = __float2half_rn(__ldcg(aq + (d ^ 64)));
            const half sn = d < 64 ? __hneg(sr[d]) : sr[d];
            gq[w * TILE + d] = __hfma(qv, cr[d], __hmul(qo, sn));
        }
        for (int i = tid; i < nseg * TILE; i += DS_CONSUMERS) {
            const int d = i & 127, sg = i >> 7, kvh = h0 + sg;
            if (!owner(kvh)) continue;
            const int plen = plen_of(kvh);
            const half* sr = BATCH ? a.sin + (size_t)plen * TILE : sr1;
            const half* cr = BATCH ? a.cos + (size_t)plen * TILE : cr1;
            const half sn = d < 64 ? __hneg(sr[d]) : sr[d];
            const float* ak = a.acc_qkv + a.HQ + (size_t)kvh * TILE;
            if constexpr (BATCH) { const int b = kvh / a.kv_heads; ak = a.acc_qkv + b * qkv_ld + a.HQ + (size_t)(kvh - b * a.kv_heads) * TILE; }
            const half kv = __float2half_rn(__ldcg(ak + d)), ko = __float2half_rn(__ldcg(ak + (d ^ 64)));
            const half kr = __hfma(kv, cr[d], __hmul(ko, sn));
            const half vv = __float2half_rn(__ldcg(BATCH ? ak + a.HKV + d : a.acc_qkv + a.HQ + a.HKV + (size_t)kvh * TILE + d));
            gkn[sg * TILE + d] = __half2float(kr); gvn[sg * TILE + d] = __half2float(vv);
            const size_t off = ((size_t)kvh * a.max_seq + plen) * TILE + d;      // cache layout q4_attn.cu:32-51, kv_heads rows (per sequence)
            L->kc[off] = kr; L->vc[off] = vv;
        }
        }
        for (int i = tid; i < nseg * nr * 4 * PART_LD; i += DS_CONSUMERS) {
            const int w = i / (4 * PART_LD), e = i - w * 4 * PART_LD;
            gparts[w * 5 * PART_LD + e] = (e % PART_LD) == 128 ? -INFINITY : 0.f;
        }
        consumer_sync();
        constexpr float LOG2E = 1.4426950408889634f;
        int u = u0 + ((wk - jbase) & 3);
        int kvh = u / nph, ch = u - kvh * nph;
        for (; u < u1; u += 4) {
            const int sg = kvh - h0;
            int nv = plen_of(kvh) - ch * 16; nv = nv < 0 ? 0 : (nv > 16 ? 16 : nv);
            const uint32_t sb = ring_a + (uint32_t)ls * STAGE_STRIDE + mbar_wait_tok(full0 + ls * 8, par, false);
            float dep = 0.f;
            for (int r = wn; r < nr && !(a.debug & 2); r += 4) {
                const uint4 qh = *reinterpret_cast<const uint4*>(gq + (sg * nr + r) * TILE + l16 * 8);
                // scores of the 16 positions: position it * 2 + sub in the lanes of half-warp sub (16 lanes x 8 dims)
                float sc[8], smax = -INFINITY;
                #pragma unroll
                for (int it = 0; it < 8; it++) {
                    const uint4 kv = lds128(sb + (uint32_t)(it * 2 + sub) * 256u + (uint32_t)l16 * 16u);
                    float d = 0.f;
                    d = fhfma2(kv.x, qh.x, d); d = fhfma2(kv.y, qh.y, d); d = fhfma2(kv.z, qh.z, d); d = fhfma2(kv.w, qh.w, d);
                    d += __shfl_xor_sync(0xffffffffu, d, 8); d += __shfl_xor_sync(0xffffffffu, d, 4);
                    d += __shfl_xor_sync(0xffffffffu, d, 2); d += __shfl_xor_sync(0xffffffffu, d, 1);
                    sc[it] = it * 2 + sub < nv ? d * scale : -INFINITY;
                    smax = fmaxf(smax, sc[it]);
                }
                smax = fmaxf(smax, __shfl_xor_sync(0xffffffffu, smax, 16));
                dep += smax;
                if (smax > -INFINITY) {
                    float* st = gparts + ((sg * nr + r) * 5 + wk) * PART_LD;
                    const float m = st[128], lsum = st[129];
                    float4 o = *reinterpret_cast<const float4*>(st + lane * 4);
                    const float mnew = fmaxf(m, smax);
                    const float alpha = ex2_ftz((m - mnew) * LOG2E);
                    float psum = 0.f;
                    #pragma unroll
                    for (int it = 0; it < 8; it++) { sc[it] = ex2_ftz((sc[it] - mnew) * LOG2E); psum += sc[it]; }
                    psum += __shfl_xor_sync(0xffffffffu, psum, 16);
                    o.x *= alpha; o.y *= alpha; o.z *= alpha; o.w *= alpha;
                    #pragma unroll
                    for (int q = 0; q < 16; q++) {
                        const float wgt = __shfl_sync(0xffffffffu, sc[q >> 1], (q & 1) * 16);
                        const uint2 vv = lds64_if(sb + 4096u + (uint32_t)q * 256u + (uint32_t)lane * 8u, q < nv);
                        const float2 f0 = __half22float2(*reinterpret_cast<const half2*>(&vv.x));
                        const float2 f1 = __half22float2(*reinterpret_cast<const half2*>(&vv.y));
                        o.x = fmaf(wgt, f0.x, o.x); o.y = fmaf(wgt, f0.y, o.y); o.z = fmaf(wgt, f1.x, o.z); o.w = fmaf(wgt, f1.y, o.w);
                    }
                    *reinterpret_cast<float4*>(st + lane * 4) = o;
                    __syncwarp();                                   // every lane has read (m, l) before lane 0 replaces them
                    if (lane == 0) { st[128] = mnew; st[129] = lsum * alpha + psum; }
                    dep += o.x;
                }
            }
            __syncwarp();
            // the arrive consumes values computed from every load of the stage: it cannot be scheduled before them
            if (lane == 0) mbar_arrive_dep(empty0 + ls * 8, dep);
            if (++ls == depth) { ls = 0; par ^= 1u; }
            ch += 4;
            while (ch >= nph) { ch -= nph; kvh++; }
        }
        // the new token (KV heads whose last chunk this CTA holds): score q . k_new, weight 1 in its own partial, per query head
        if constexpr (MULTI) {
            // token t's causal tail: an online-softmax partial over the new rows 0 .. t of the launch (t == 0: exactly the single token's)
            for (int w = warp; w < nseg * nr; w += DS_NCW) {
                const int sg = w / nr, t = (w - sg * nr) / a.n_rep;
                if (!owner(h0 + sg)) continue;
                float m = -INFINITY, lsum = 0.f;
                float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
                for (int j = 0; j <= t; j++) {
                    const float* kr = gkn + (sg * nt + j) * TILE + lane * 4;
                    float d = 0.f;
                    #pragma unroll
                    for (int c = 0; c < 4; c++) d = fmaf(__half2float(gq[w * TILE + lane * 4 + c]) * scale, kr[c], d);
                    #pragma unroll
                    for (int off = 16; off > 0; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
                    const float mnew = fmaxf(m, d);
                    const float alpha = __expf(m - mnew), pj = __expf(d - mnew);
                    const float4 v = *reinterpret_cast<const float4*>(gvn + (sg * nt + j) * TILE + lane * 4);
                    o.x = fmaf(pj, v.x, o.x * alpha); o.y = fmaf(pj, v.y, o.y * alpha); o.z = fmaf(pj, v.z, o.z * alpha); o.w = fmaf(pj, v.w, o.w * alpha);
                    lsum = fmaf(lsum, alpha, pj);
                    m = mnew;
                }
                float* pw = gparts + (w * 5 + 4) * PART_LD;
                *reinterpret_cast<float4*>(pw + lane * 4) = o;
                if (lane == 0) { pw[128] = m; pw[129] = lsum; }
            }
        } else {
        for (int w = warp; w < nseg * nr; w += DS_NCW) {
            const int sg = w / nr;
            if (!owner(h0 + sg)) continue;
            float d = 0.f;
            #pragma unroll
            for (int c = 0; c < 4; c++) d = fmaf(__half2float(gq[w * TILE + lane * 4 + c]) * scale, gkn[sg * TILE + lane * 4 + c], d);
            #pragma unroll
            for (int off = 16; off > 0; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
            float* pw = gparts + (w * 5 + 4) * PART_LD;
            *reinterpret_cast<float4*>(pw + lane * 4) = *reinterpret_cast<const float4*>(gvn + sg * TILE + lane * 4);
            if (lane == 0) { pw[128] = d; pw[129] = 1.0f; }
        }
        }
        consumer_sync();
        // this CTA's partial of every query head of its segments -> its slot of the head's CTA range
        for (int i = tid; i < nseg * nr * TILE; i += DS_CONSUMERS) {
            const int d = i & 127, w = i >> 7, sg = w / nr, h = (h0 + sg) * nr + (w - sg * nr);
            const float* pp = gparts + w * 5 * PART_LD;
            const int np = owner(h0 + sg) ? 5 : 4;
            float M = -INFINITY;
            for (int k = 0; k < np; k++) M = fmaxf(M, pp[k * PART_LD + 128]);
            float Lt = 0.f, ov = 0.f;
            for (int k = 0; k < np; k++) {
                const float mw = pp[k * PART_LD + 128];
                const float wgt = mw == -INFINITY ? 0.f : __expf(mw - M);
                Lt = fmaf(pp[k * PART_LD + 129], wgt, Lt);
                ov = fmaf(pp[k * PART_LD + d], wgt, ov);
            }
            // MULTI: query vector j = t * n_rep + r of the segment is virtual query head t * heads + (KV head) * n_rep + r
            const int hv = MULTI ? ((w - sg * nr) / a.n_rep) * a.heads + (h0 + sg) * a.n_rep + (w - sg * nr) % a.n_rep : h;
            float* dst = a.att_part + ((size_t)hv * a.att_slots + (cta - (int)s_clo[hv])) * PART_LD;
            dst[d] = ov;
            if (d == 0) { dst[128] = M; dst[129] = Lt; }
        }
    };

    #pragma unroll 1
    for (int l = 0; l < a.n_layers; l++) {
        const LayerDesc* L = a.layers + l;
        // ======================================================== QKV ========================================================
        {
            const Phase p = phase_of(a, PH_QKV, G, nb);
            const int u0 = s_rng[PH_QKV][0], u1 = s_rng[PH_QKV][1];
            stamp(l, 0);
            if (l > 0) zero_share(a.acc_gu, ZR_GU);
            residual_and_norm(l > 0 ? a.acc_d : nullptr, (TP && !a.tp_reduce && l > 0) ? a.slots_d : nullptr, epoch0 + 2u * (l - 1) + 1u);
            stamp(l, 15);
            if constexpr (!ACT) { if (u1 > u0) for (int b = 0; b < nb; b++) stage_xd(s_rng[p.kind][2], s_rng[p.kind][3], p.spt, norm_get(b, rm_of(b)), b); }
            else stage_phase(p, u0, u1, [&](int m) { return norm_get_map(L->ln1, rm_of(0), L->xmap[m]); });
            consumer_sync();
            if constexpr (LORA) {
                if (lora_a(l, p, [&](int b) { return lora_norm_get(L->ln1, b, rm_of(b)); })) grid_barrier(a.bar, target, (unsigned)G, tid);
            }
            stamp(l, 1);
            gemv(p, u0, u1);
            if constexpr (LORA) lora_b(l, p, u0, u1);
            jbase += u1 - u0;
            stamp(l, 2);
        }
        grid_barrier(a.bar, target, (unsigned)G, tid, &s_arrived);
        stamp(l, 3);

        // ======================================================== ATT ========================================================
        {
            const Phase p = step_phase<MULTI>(a, PH_ATT, G, nb);
            const int u0 = s_rng[PH_ATT][0], u1 = s_rng[PH_ATT][1];
            if (l > 0) zero_share(a.acc_d, ZR_H);
            const int nph = p.tpm;
            const float scale = rsqrtf((float)TILE);
            const int l16 = lane & 15, sub = lane >> 4;
            const int h0 = u1 > u0 ? u0 / nph : 0;
            const int nseg = u1 > u0 ? (u1 - 1) / nph - h0 + 1 : 0;            // <= 2 (heads <= grid: exl_decode_plan_create checks it against the plan's grid)
            if constexpr (GQA || MULTI) att_gqa(L, u0, u1, nph, h0, nseg);
            else {
                // every segment's q (and the new k / v rows where this CTA owns the head's last chunk): one L2 round trip
                if (tid < nseg * TILE) {
                    const int sg = tid >> 7, d = tid & 127, h = h0 + sg;
                    const bool owner = min(u1, (h + 1) * nph) == (h + 1) * nph;
                    // BATCH: h is the virtual head b * heads + hl -- sequence b's context and accumulator row
                    int plen = a.past_len, hl = h; size_t qb = 0;
                    if constexpr (BATCH) { const int b = h / a.heads; plen = a.past_lens[b]; hl = h - b * a.heads; qb = (size_t)b * (a.HQ + 2 * a.HKV); }
                    // fp16 projection result, rope in fp16 with the reference's instruction order (rope.cu:48-67)
                    const half* sr = a.sin + (size_t)plen * TILE;
                    const half* cr = a.cos + (size_t)plen * TILE;
                    const float* aq = a.acc_qkv + qb + (size_t)hl * TILE;
                    const half qv = __float2half_rn(__ldcg(aq + d)), qo = __float2half_rn(__ldcg(aq + (d ^ 64)));
                    const half sn = d < 64 ? __hneg(sr[d]) : sr[d];
                    const half qr = __hfma(qv, cr[d], __hmul(qo, sn));
                    qh_s[sg * TILE + d] = qr;
                    q_s[sg * TILE + d] = __half2float(qr) * scale;
                    if (owner) {
                        const float* ak = a.acc_qkv + qb + a.HQ + (size_t)hl * TILE;
                        const half kv = __float2half_rn(__ldcg(ak + d)), ko = __float2half_rn(__ldcg(ak + (d ^ 64)));
                        const half kr = __hfma(kv, cr[d], __hmul(ko, sn));
                        const half vv = __float2half_rn(__ldcg(a.acc_qkv + qb + 2 * a.HQ + (size_t)hl * TILE + d));
                        kn_s[sg * TILE + d] = __half2float(kr); vn_s[sg * TILE + d] = __half2float(vv);
                        const size_t off = ((size_t)h * a.max_seq + plen) * TILE + d;      // cache layout q4_attn.cu:32-51
                        L->kc[off] = kr; L->vc[off] = vv;
                    }
                }
                consumer_sync();
                {
                    // this pipeline's stages, in order; the 4 warps of the pipeline take 4 positions of each 16-position chunk
                    uint4 qh = make_uint4(0u, 0u, 0u, 0u);          // 8 fp16 q values of this lane's dims
                    float m = -INFINITY, lsum = 0.f, o[4] = {0.f, 0.f, 0.f, 0.f};
                    int cur = -1;                                  // segment the running (m, l, o) belongs to
                    auto put_part = [&]() {
                        float* pw = parts + (cur * 17 + warp) * PART_LD;
                        *reinterpret_cast<float4*>(pw + lane * 4) = make_float4(o[0], o[1], o[2], o[3]);
                        if (lane == 0) { pw[128] = m; pw[129] = lsum; }
                    };
                    int u = u0 + ((wk - jbase) & 3);
                    int h = u / nph, ch = u - h * nph;             // (head, chunk) of the unit, advanced without divisions
                    // 32-bit shared addresses from per-lane constants, as in the GEMV loop: K row of position wn * 4 + it * 2 + sub (16 lanes x
                    // 16 B), V row of position wn * 4 + q (32 lanes x 8 B)
                    const uint32_t k_lane = (uint32_t)((wn * 4 + sub) * 256 + l16 * 16);
                    const uint32_t v_lane = (uint32_t)(4096 + wn * 4 * 256 + lane * 8);
                    constexpr float LOG2E = 1.4426950408889634f;
                    for (; u < u1; u += 4) {
                        const int sg = h - h0;
                        if (sg != cur) {
                            if (cur >= 0) put_part();
                            cur = sg; m = -INFINITY; lsum = 0.f; o[0] = o[1] = o[2] = o[3] = 0.f;
                            qh = *reinterpret_cast<const uint4*>(qh_s + sg * TILE + l16 * 8);
                        }
                        int plen = a.past_len;
                        if constexpr (BATCH) plen = a.past_lens[h / a.kv_heads];
                        int nv = plen - ch * 16; nv = nv < 0 ? 0 : (nv > 16 ? 16 : nv);
                        // the zero token ties the (freely schedulable) asm loads below to the wait
                        const uint32_t sb = ring_a + (uint32_t)ls * STAGE_STRIDE + mbar_wait_tok(full0 + ls * 8, par, false);
                        float sc2[2];
                        float smax = -INFINITY;
                        #pragma unroll
                        for (int it = 0; it < 2; it++) {
                            const int pp = wn * 4 + it * 2 + sub;
                            const uint4 kv = lds128(sb + k_lane + it * 512);
                            float d = 0.f;
                            d = fhfma2(kv.x, qh.x, d); d = fhfma2(kv.y, qh.y, d); d = fhfma2(kv.z, qh.z, d); d = fhfma2(kv.w, qh.w, d);
                            d += __shfl_xor_sync(0xffffffffu, d, 8); d += __shfl_xor_sync(0xffffffffu, d, 4);
                            d += __shfl_xor_sync(0xffffffffu, d, 2); d += __shfl_xor_sync(0xffffffffu, d, 1);
                            sc2[it] = pp < nv ? d * scale : -INFINITY;
                            smax = fmaxf(smax, sc2[it]);
                        }
                        smax = fmaxf(smax, __shfl_xor_sync(0xffffffffu, smax, 16));
                        if (smax > -INFINITY && !(a.debug & 2)) {           // this warp has at least one valid position in the chunk
                            const float mnew = fmaxf(m, smax);
                            const float alpha = ex2_ftz((m - mnew) * LOG2E);
                            sc2[0] = ex2_ftz((sc2[0] - mnew) * LOG2E); sc2[1] = ex2_ftz((sc2[1] - mnew) * LOG2E);
                            float psum = sc2[0] + sc2[1];
                            psum += __shfl_xor_sync(0xffffffffu, psum, 16);
                            lsum = lsum * alpha + psum;
                            #pragma unroll
                            for (int c = 0; c < 4; c++) o[c] *= alpha;
                            m = mnew;
                            #pragma unroll
                            for (int q = 0; q < 4; q++) {
                                // positions past the context end: weight 0 (their score is -inf) times a row that is not loaded (zeros)
                                const float wgt = __shfl_sync(0xffffffffu, sc2[q >> 1], (q & 1) * 16);
                                const uint2 vv = lds64_if(sb + v_lane + q * 256, wn * 4 + q < nv);
                                const float2 f0 = __half22float2(*reinterpret_cast<const half2*>(&vv.x));
                                const float2 f1 = __half22float2(*reinterpret_cast<const half2*>(&vv.y));
                                o[0] = fmaf(wgt, f0.x, o[0]); o[1] = fmaf(wgt, f0.y, o[1]); o[2] = fmaf(wgt, f1.x, o[2]); o[3] = fmaf(wgt, f1.y, o[3]);
                            }
                        }
                        __syncwarp();
                        // the arrive consumes values computed from every load of the stage: it cannot be scheduled before them
                        if (lane == 0) mbar_arrive_dep(empty0 + ls * 8, o[0] + smax);
                        if (++ls == depth) { ls = 0; par ^= 1u; }
                        ch += 4;
                        while (ch >= nph) { ch -= nph; h++; }
                    }
                    if (cur >= 0) put_part();
                    // segments this warp saw no stage of: an empty partial
                    for (int sg = 0; sg < nseg; sg++) {
                        const int first = max(u0, (h0 + sg) * nph), last = min(u1, (h0 + sg + 1) * nph);
                        // did this pipeline get a stage of segment sg?  stages of the segment: local indices [first - u0, last - u0)
                        const int i0 = (first - u0) + ((wk - (jbase + (first - u0))) & 3);
                        if (i0 >= last - u0) {
                            float* pw = parts + (sg * 17 + warp) * PART_LD;
                            *reinterpret_cast<float4*>(pw + lane * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
                            if (lane == 0) { pw[128] = -INFINITY; pw[129] = 0.f; }
                        }
                    }
                    if (warp < nseg) {
                        // the new token itself (segments whose last chunk this CTA holds): score q . k_new, weight 1 in its own partial
                        const int sg = warp, h = h0 + sg;
                        if (min(u1, (h + 1) * nph) == (h + 1) * nph) {
                            float d = 0.f;
                            #pragma unroll
                            for (int c = 0; c < 4; c++) d = fmaf(q_s[sg * TILE + lane * 4 + c], kn_s[sg * TILE + lane * 4 + c], d);
                            #pragma unroll
                            for (int off = 16; off > 0; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
                            float* pw = parts + (sg * 17 + 16) * PART_LD;
                            *reinterpret_cast<float4*>(pw + lane * 4) = *reinterpret_cast<const float4*>(vn_s + sg * TILE + lane * 4);
                            if (lane == 0) { pw[128] = d; pw[129] = 1.0f; }
                        }
                    }
                }
                consumer_sync();
                if (tid < nseg * TILE) {
                    const int sg = tid >> 7, d = tid & 127, h = h0 + sg;
                    const bool owner = min(u1, (h + 1) * nph) == (h + 1) * nph;
                    const float* pp = parts + sg * 17 * PART_LD;
                    const int np = owner ? 17 : 16;
                    float M = -INFINITY;
                    for (int w = 0; w < np; w++) M = fmaxf(M, pp[w * PART_LD + 128]);
                    float Lt = 0.f, ov = 0.f;
                    for (int w = 0; w < np; w++) {
                        const float mw = pp[w * PART_LD + 128];
                        const float wgt = mw == -INFINITY ? 0.f : __expf(mw - M);
                        Lt = fmaf(pp[w * PART_LD + 129], wgt, Lt);
                        ov = fmaf(pp[w * PART_LD + d], wgt, ov);
                    }
                    const int slot_id = cta - (int)s_clo[h];
                    float* dst = a.att_part + ((size_t)h * a.att_slots + slot_id) * PART_LD;
                    dst[d] = ov;
                    if (d == 0) { dst[128] = M; dst[129] = Lt; }
                }
            }
            jbase += u1 - u0;
            stamp(l, 4);
        }
        grid_barrier(a.bar, target, (unsigned)G, tid, &s_arrived);
        stamp(l, 5);

        // ========================================================= O =========================================================
        {
            const Phase p = phase_of(a, PH_O, G, nb);
            const int u0 = s_rng[PH_O][0], u1 = s_rng[PH_O][1];
            zero_share(a.acc_qkv, ZR_QKV);
            // softmax-combine of the CTA partials of one head (model.py:402-409), 8 dims per thread, fp16 result.
            // All loads of up to 4 partials per round are issued together: one L2 round trip per round.
            auto combine8 = [&](int h, int d0) -> uint4 {
                const int ns = (int)s_chi[h] - (int)s_clo[h] + 1;
                const float* src = a.att_part + (size_t)h * a.att_slots * PART_LD;
                float Lt = 0.f, ov[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, M = -INFINITY;
                for (int b = 0; b < ns; b += 4) {
                    float mw[4], lw[4]; float4 o0[4], o1[4];
                    #pragma unroll
                    for (int q = 0; q < 4; q++) {
                        const bool ok = b + q < ns;
                        const float* sp = src + (size_t)(ok ? b + q : 0) * PART_LD;
                        mw[q] = ok ? __ldcg(sp + 128) : -INFINITY; lw[q] = __ldcg(sp + 129);
                        o0[q] = ldcg4(sp + d0); o1[q] = ldcg4(sp + d0 + 4);
                    }
                    float Mn = M;
                    #pragma unroll
                    for (int q = 0; q < 4; q++) Mn = fmaxf(Mn, mw[q]);
                    const float resc = M == -INFINITY ? 0.f : __expf(M - Mn);
                    Lt *= resc;
                    #pragma unroll
                    for (int i = 0; i < 8; i++) ov[i] *= resc;
                    M = Mn;
                    #pragma unroll
                    for (int q = 0; q < 4; q++) {
                        const float wgt = mw[q] == -INFINITY ? 0.f : __expf(mw[q] - M);
                        Lt = fmaf(lw[q], wgt, Lt);
                        ov[0] = fmaf(o0[q].x, wgt, ov[0]); ov[1] = fmaf(o0[q].y, wgt, ov[1]); ov[2] = fmaf(o0[q].z, wgt, ov[2]); ov[3] = fmaf(o0[q].w, wgt, ov[3]);
                        ov[4] = fmaf(o1[q].x, wgt, ov[4]); ov[5] = fmaf(o1[q].y, wgt, ov[5]); ov[6] = fmaf(o1[q].z, wgt, ov[6]); ov[7] = fmaf(o1[q].w, wgt, ov[7]);
                    }
                }
                const float inv = 1.0f / Lt;
                uint4 r; half2* hh = reinterpret_cast<half2*>(&r);
                #pragma unroll
                for (int i = 0; i < 4; i++) hh[i] = __floats2half2_rn(ov[2 * i] * inv, ov[2 * i + 1] * inv);
                return r;
            };
            if constexpr (!ACT) {
                // stage k of sequence b's o_proj input is virtual head b * heads + k: the CTA combines exactly the heads its K range needs
                if (u1 > u0)
                    for (int b = 0; b < nb; b++)
                        stage_xd(s_rng[PH_O][2], s_rng[PH_O][3], p.spt, [&](int k8, int) -> uint4 { return combine8(b * a.heads + (k8 >> 4), (k8 & 15) * 8); }, b);
            } else {
                // act-order o_proj: its input is a gather over ALL heads (x_map), so the combined attention output is first written
                // to L2 once (head h by CTA h mod grid), one extra grid barrier, then every CTA gathers what its K range needs
                for (int h = cta; h < a.heads; h += G)
                    if (tid < 16) reinterpret_cast<uint4*>(a.attn_vec + (size_t)h * TILE)[tid] = combine8(h, tid * 8);
                grid_barrier(a.bar, target, (unsigned)G, tid);
                const uint32_t* map = L->xmap[3];
                stage_phase(p, u0, u1, [&](int) {
                    return [=](int k8, int) -> uint4 {
                        uint32_t idx[8];
                        load_map8(map, k8, idx);
                        uint4 r; half* hh = reinterpret_cast<half*>(&r);
                        #pragma unroll
                        for (int i = 0; i < 8; i++) hh[i] = __ushort_as_half(__ldcg(reinterpret_cast<const unsigned short*>(a.attn_vec) + idx[i]));
                        return r;
                    };
                });
            }
            consumer_sync();
            if constexpr (LORA) {
                // un-gathered o_proj input: act-order has it in attn_vec already, otherwise the softmax-combine yields it
                bool adapted;
                if constexpr (ACT) adapted = lora_a(l, p, [&](int) { return [&](int k8) -> uint4 { return __ldcg(reinterpret_cast<const uint4*>(a.attn_vec) + k8); }; });
                else adapted = lora_a(l, p, [&](int b) { return [&, b](int k8) -> uint4 { return combine8(b * a.heads + (k8 >> 4), (k8 & 15) * 8); }; });
                if (adapted) grid_barrier(a.bar, target, (unsigned)G, tid);
            }
            stamp(l, 6);
            gemv(p, u0, u1);
            if constexpr (LORA) lora_b(l, p, u0, u1);
            jbase += u1 - u0;
            preload_norm(L->ln2, phase_of(a, PH_GU, G, nb));
            stamp(l, 7);
        }
        if constexpr (TP) push_partial(a.acc_o, a.push_o, epoch0 + 2u * l, l, 16);
        else grid_barrier(a.bar, target, (unsigned)G, tid, &s_arrived);
        stamp(l, 8);

        // ========================================================= GU ========================================================
        {
            const Phase p = phase_of(a, PH_GU, G, nb);
            const int u0 = s_rng[PH_GU][0], u1 = s_rng[PH_GU][1];
            residual_and_norm(a.acc_o, (TP && !a.tp_reduce) ? a.slots_o : nullptr, epoch0 + 2u * l);
            if constexpr (!ACT) { if (u1 > u0) for (int b = 0; b < nb; b++) stage_xd(s_rng[p.kind][2], s_rng[p.kind][3], p.spt, norm_get(b, rm_of(b)), b); }
            else stage_phase(p, u0, u1, [&](int m) { return norm_get_map(L->ln2, rm_of(0), L->xmap[m]); });
            consumer_sync();
            if constexpr (LORA) {
                if (lora_a(l, p, [&](int b) { return lora_norm_get(L->ln2, b, rm_of(b)); })) grid_barrier(a.bar, target, (unsigned)G, tid);
            }
            stamp(l, 9);
            gemv(p, u0, u1);
            if constexpr (LORA) lora_b(l, p, u0, u1);
            jbase += u1 - u0;
            stamp(l, 10);
        }
        grid_barrier(a.bar, target, (unsigned)G, tid, &s_arrived);
        stamp(l, 11);

        // ======================================================== DOWN =======================================================
        {
            const Phase p = phase_of(a, PH_DOWN, G, nb);
            const int u0 = s_rng[PH_DOWN][0], u1 = s_rng[PH_DOWN][1];
            zero_share(a.acc_o, ZR_H);
            if constexpr (!ACT) {
                // BATCH: sequence b reads its own [gate | up] row of the accumulator
                if (u1 > u0) for (int b = 0; b < nb; b++) stage_xd(s_rng[PH_DOWN][2], s_rng[PH_DOWN][3], p.spt, [&](int k8, int) -> uint4 {
                    // silu(gate) * up on the fp16-rounded projections (q4_mlp.cu:27-36,46-88)
                    const float* gu = a.acc_gu + (size_t)b * 2 * a.I;
                    const float4 g0 = ldcg4(gu + k8 * 8), g1 = ldcg4(gu + k8 * 8 + 4);
                    const float4 u0v = ldcg4(gu + a.I + k8 * 8), u1v = ldcg4(gu + a.I + k8 * 8 + 4);
                    const float gf[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
                    const float uf[8] = {u0v.x, u0v.y, u0v.z, u0v.w, u1v.x, u1v.y, u1v.z, u1v.w};
                    uint4 r; half* hh = reinterpret_cast<half*>(&r);
                    #pragma unroll
                    for (int i = 0; i < 8; i++) hh[i] = __hmul(silu_h(__float2half_rn(gf[i])), __float2half_rn(uf[i]));
                    return r;
                }, b);
            } else {
                const uint32_t* map = L->xmap[6];
                stage_phase(p, u0, u1, [&](int) {
                    return [=](int k8, int) -> uint4 {
                        uint32_t idx[8];
                        load_map8(map, k8, idx);
                        uint4 r; half* hh = reinterpret_cast<half*>(&r);
                        #pragma unroll
                        for (int i = 0; i < 8; i++)
                            hh[i] = __hmul(silu_h(__float2half_rn(__ldcg(a.acc_gu + idx[i]))), __float2half_rn(__ldcg(a.acc_gu + a.I + idx[i])));
                        return r;
                    };
                });
            }
            consumer_sync();
            if constexpr (LORA) {
                // silu(gate) * up of sequence b, un-gathered
                auto act_get = [&](int b) {
                    return [&, b](int k8) -> uint4 {
                        const float* gu = a.acc_gu + (size_t)b * 2 * a.I;
                        uint4 r; half* hh = reinterpret_cast<half*>(&r);
                        #pragma unroll
                        for (int i = 0; i < 8; i++) hh[i] = __hmul(silu_h(__float2half_rn(__ldcg(gu + k8 * 8 + i))), __float2half_rn(__ldcg(gu + a.I + k8 * 8 + i)));
                        return r;
                    };
                };
                if (lora_a(l, p, act_get)) grid_barrier(a.bar, target, (unsigned)G, tid);
            }
            stamp(l, 12);
            gemv(p, u0, u1);
            if constexpr (LORA) lora_b(l, p, u0, u1);
            jbase += u1 - u0;
            if (l + 1 < a.n_layers) preload_norm(a.layers[l + 1].ln1, phase_of(a, PH_QKV, G, nb));
            stamp(l, 13);
        }
        if constexpr (TP) push_partial(a.acc_d, a.push_d, epoch0 + 2u * l + 1u, l, 18);
        else grid_barrier(a.bar, target, (unsigned)G, tid, &s_arrived);
        stamp(l, 14);
    }

    // ========================================================= HEAD ==========================================================
    residual_and_norm(a.n_layers > 0 ? a.acc_d : nullptr, (TP && !a.tp_reduce && a.n_layers > 0) ? a.slots_d : nullptr, epoch0 + 2u * (a.n_layers - 1) + 1u);
    if (a.x_out && cta == 0)
        for (int i = tid; i < nb * a.H / 8; i += DS_CONSUMERS) reinterpret_cast<uint4*>(a.x_out)[i] = reinterpret_cast<const uint4*>(xres)[i];
    if (a.lm_head) {
        const int u0 = s_rng[PH_HEAD][0], u1 = s_rng[PH_HEAD][1];
        const int h8 = a.H / 8;
        for (int b = 0; b < nb; b++) {
            const half2 rm2 = __float2half2_rn(rm_of(b));
            for (int j = tid; j < h8; j += DS_CONSUMERS) {
                uint4 xv = reinterpret_cast<const uint4*>(xres)[b * h8 + j];
                const uint4 wv = __ldg(reinterpret_cast<const uint4*>(a.final_norm) + j);
                half2* h = reinterpret_cast<half2*>(&xv); const half2* w2 = reinterpret_cast<const half2*>(&wv);
                #pragma unroll
                for (int q = 0; q < 4; q++) h[q] = __hmul2(__hmul2(h[q], rm2), w2[q]);
                reinterpret_cast<uint4*>(xh)[b * h8 + j] = xv;
            }
        }
        consumer_sync();
        // stage = 8 chunks of 512 fp16 of the row-major [vocab, H] matrix; the 4 warps of the pipeline take 2 chunks each and dot
        // every chunk with every sequence's normalised x
        const int cpr = a.H >> 9;                               // chunks per vocabulary row
        const long long nchunks = (long long)a.vocab * cpr;
        for (int u = u0 + ((wk - jbase) & 3); u < u1; u += 4) {
            mbar_wait(full0 + ls * 8, par);
            const unsigned char* sb = ring + (size_t)(wk * depth + ls) * STAGE_STRIDE;
            const long long c0 = (long long)u * 8 + wn * 2;
            long long row = c0 / cpr; int kc = (int)(c0 - row * cpr);
            float part[MAX_BATCH] = {0.f, 0.f, 0.f, 0.f};
            #pragma unroll 1
            for (int cc = 0; cc < ((a.debug & 4) ? 0 : 2) && c0 + cc < nchunks; cc++) {
                #pragma unroll
                for (int hf = 0; hf < 2; hf++) {
                    const uint4 wv = *reinterpret_cast<const uint4*>(sb + (wn * 2 + cc) * 1024 + hf * 512 + lane * 16);
                    #pragma unroll
                    for (int b = 0; b < MAX_BATCH; b++) {
                        if (b < nb) {
                            const uint4 xv = *reinterpret_cast<const uint4*>(reinterpret_cast<const unsigned char*>(xh + (size_t)b * a.H) + (size_t)kc * 1024 + hf * 512 + lane * 16);
                            part[b] = fhfma2(wv.x, xv.x, part[b]); part[b] = fhfma2(wv.y, xv.y, part[b]);
                            part[b] = fhfma2(wv.z, xv.z, part[b]); part[b] = fhfma2(wv.w, xv.w, part[b]);
                        }
                    }
                }
                if (++kc == cpr || cc == 1 || c0 + cc + 1 == nchunks) {
                    #pragma unroll
                    for (int b = 0; b < MAX_BATCH; b++) {
                        if (b < nb) {
                            float tot = part[b];
                            #pragma unroll
                            for (int off = 16; off > 0; off >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, off);
                            if (lane == 0) atomicAdd(a.logits + (size_t)b * a.vocab + row, tot);
                        }
                        part[b] = 0.f;
                    }
                    if (kc == cpr) { kc = 0; row++; }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty0 + ls * 8);
            if (++ls == depth) { ls = 0; par ^= 1u; }
        }
    }
}

// Attention partial table -> neutral partials (o = 0, m = -inf, l = 0).  Launched by exl_decode_step before a step whose attention
// phase leaves CTAs idle inside a head's CTA range (short contexts, decode_step_sched.h: att_needs_reset): the slots those CTAs would
// have written must not carry partials of an earlier, longer context into the O prologue's combine.
__global__ void att_part_reset_kernel(float* __restrict__ att_part, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) att_part[i] = (i % PART_LD) == 128 ? -INFINITY : 0.f;
}

} // namespace

// ---------------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------------
struct exl_decode_plan
{
    int device = 0;
    StepArgs args;
    LayerDesc* d_layers = nullptr;
    unsigned char* d_scratch = nullptr;
    unsigned char* d_shared = nullptr;          // {slots_o[world][H], slots_d[world][H]} of {value, epoch} pairs: the part peers map through cudaIpc
    size_t shared_o = 0, shared_d = 0, shared_bar = 0;
    unsigned char* peer_base[8] = {nullptr};    // mapped peer regions (own entry == d_shared)
    bool peers_ready = false;
    size_t smem = 0;
    int grid = 0;
    int max_batch = 1;                          // sequences a step may carry (> 1: the BATCH kernels)
    LoraMat* d_lora = nullptr;                  // LoRA plans (the LORA kernels): [n_layers * 7] adapters
    long long lora_barriers = 0;                // their extra grid barriers per step
    int max_tokens = 0;                         // multi-token plans (the MULTI kernel): tokens of one sequence a step may carry; else 0
    int cache_seqs = 0;                         // multi-token plans: sequences the caches hold
};

// the one multi-token instantiation: batch GEMVs and head, the grouped-query attention path for any n_rep
static const void* multi_kernel() { return (const void*)decode_step_kernel<false, false, true, true, false, true>; }

static const void* step_kernel_for(bool act, bool tp, bool gqa, bool batch, bool lora = false)
{
    if (lora) {                                                                     // never under TP; a batch without act-order
        if (batch) return gqa ? (const void*)decode_step_kernel<false, false, true, true, true> : (const void*)decode_step_kernel<false, false, false, true, true>;
        if (gqa) return act ? (const void*)decode_step_kernel<true, false, true, false, true> : (const void*)decode_step_kernel<false, false, true, false, true>;
        return act ? (const void*)decode_step_kernel<true, false, false, false, true> : (const void*)decode_step_kernel<false, false, false, false, true>;
    }
    if (batch) return gqa ? (const void*)decode_step_kernel<false, false, true, true> : (const void*)decode_step_kernel<false, false, false, true>;   // neither act-order nor TP
    if (gqa) return act ? (const void*)decode_step_kernel<true, false, true, false> : (const void*)decode_step_kernel<false, false, true, false>;     // no GQA under TP
    if (act) return tp ? (const void*)decode_step_kernel<true, true, false, false> : (const void*)decode_step_kernel<true, false, false, false>;
    return tp ? (const void*)decode_step_kernel<false, true, false, false> : (const void*)decode_step_kernel<false, false, false, false>;
}

static int plan_fail(exl_decode_plan* p, int rc)
{
    if (p) {
        for (int r = 0; r < 8; r++) if (p->peer_base[r] && p->peer_base[r] != p->d_shared) cudaIpcCloseMemHandle(p->peer_base[r]);
        if (p->d_layers) cudaFree(p->d_layers);
        if (p->d_scratch) cudaFree(p->d_scratch);
        if (p->d_shared) cudaFree(p->d_shared);
        if (p->d_lora) cudaFree(p->d_lora);
        delete p;
    }
    return rc;
}

extern "C" int exl_decode_plan_create(const exl_decode_desc* d, exl_decode_plan** out)
{
    return exl_decode_plan_create_batch(d, 1, out);
}

static int plan_create(const exl_decode_desc* d, int max_batch, const exl_decode_lora* lora, exl_decode_plan** out, int max_tokens = 0,
                       int cache_seqs = 0);

extern "C" int exl_decode_plan_create_batch(const exl_decode_desc* d, int max_batch, exl_decode_plan** out)
{
    return plan_create(d, max_batch, nullptr, out);
}

extern "C" int exl_decode_plan_create_multi(const exl_decode_desc* d, int max_tokens, int cache_seqs, exl_decode_plan** out)
{
    if (!d || !out) return exl_set_err(EXL_ERR_ARG, "decode_plan_multi: NULL argument");
    *out = nullptr;
    if (max_tokens < 1 || max_tokens > MAX_BATCH)
        return exl_set_err(EXL_ERR_ARG, "decode_plan_multi: max_tokens %d outside 1..%d: run longer chunks through prefill", max_tokens, MAX_BATCH);
    if (d->tp_world > 1)
        return exl_set_err(EXL_ERR_ARG, "decode_plan_multi: tensor parallelism (world %d) is not supported by the multi-token step: use exl_decode_step per token or prefill", d->tp_world);
    if (cache_seqs < 1)
        return exl_set_err(EXL_ERR_ARG, "decode_plan_multi: cache_seqs %d: the caches must hold at least 1 sequence", cache_seqs);
    return plan_create(d, max_tokens, nullptr, out, max_tokens, cache_seqs);
}

extern "C" int exl_decode_plan_create_lora(const exl_decode_desc* d, int max_batch, const exl_decode_lora* lora, exl_decode_plan** out)
{
    if (!d || !out) return exl_set_err(EXL_ERR_ARG, "decode_plan: NULL argument");
    if (!lora) return plan_create(d, max_batch, nullptr, out);
    *out = nullptr;
    if (lora->n_layers != d->n_layers)
        return exl_set_err(EXL_ERR_ARG, "decode_plan_lora: the adapter has %d layers, the model %d: give one entry per layer (rank 0 where there is none)", lora->n_layers, d->n_layers);
    if (d->n_layers < 1 || d->n_layers > MAX_LAYERS || !lora->rank) return exl_set_err(EXL_ERR_ARG, "decode_plan_lora: bad layer count %d or NULL rank array", d->n_layers);
    bool any = false;
    for (int i = 0; i < 7 * d->n_layers; i++) any = any || lora->rank[i] != 0;
    if (!any) return plan_create(d, max_batch, nullptr, out);                  // no adapter: exactly the plan without one
    if (d->tp_world > 1)
        return exl_set_err(EXL_ERR_ARG, "decode_plan_lora: LoRA adapters under tensor parallelism are not supported by the fused step: use the per-op path");
    if (!lora->a || !lora->b) return exl_set_err(EXL_ERR_ARG, "decode_plan_lora: NULL A or B array: use the per-op path for this adapter");
    for (int i = 0; i < 7 * d->n_layers; i++) {
        const int r = lora->rank[i], l = i / 7, m = i % 7;
        if (r == 0) continue;
        if (!lora_rank_ok(r))
            return exl_set_err(EXL_ERR_ARG, "decode_plan_lora: layer %d matrix %d has rank %d; the fused step takes multiples of 8 up to %d: use the per-op path", l, m, r, LORA_MAX_RANK);
        if (!lora->a[i] || !lora->b[i])
            return exl_set_err(EXL_ERR_ARG, "decode_plan_lora: layer %d matrix %d has rank %d but a NULL A or B: use the per-op path", l, m, r);
        if (((uintptr_t)lora->a[i] | (uintptr_t)lora->b[i]) & 15)
            return exl_set_err(EXL_ERR_ARG, "decode_plan_lora: layer %d matrix %d: A and B must be 16-byte aligned for the fused step: use the per-op path", l, m);
    }
    return plan_create(d, max_batch, lora, out);
}

static int plan_create(const exl_decode_desc* d, int max_batch, const exl_decode_lora* lora, exl_decode_plan** out, int max_tokens,
                       int cache_seqs)
{
    const bool multi = max_tokens > 0;                 // max_batch == max_tokens then: accumulator rows and virtual heads per token
    if (!d || !out) return exl_set_err(EXL_ERR_ARG, "decode_plan: NULL argument");
    *out = nullptr;
    if (max_batch < 1 || max_batch > MAX_BATCH)
        return exl_set_err(EXL_ERR_ARG, "decode_plan: max_batch %d outside 1..%d: step larger batches in groups of up to %d sequences or use the per-op path", max_batch, MAX_BATCH, MAX_BATCH);
    if (d->n_layers < 1 || d->n_layers > MAX_LAYERS || !d->mats || !d->mats[0]) return exl_set_err(EXL_ERR_ARG, "decode_plan: bad layer count %d", d->n_layers);
    const exl_q4_matrix* q0 = d->mats[0];
    ExlDevice* ds = exl_device_state(q0->device);
    if (!ds) return EXL_ERR_CUDA;
    DeviceGuard guard(q0->device);
    const int H = q0->K, HQ = q0->N, I = d->mats[4]->N;
    if (d->head_dim != TILE || d->num_heads * TILE != HQ) return exl_set_err(EXL_ERR_ARG, "decode_plan: head_dim must be 128 and heads * 128 == q_proj width (%d heads, width %d)", d->num_heads, HQ);
    const int kv_heads = d->num_kv_heads ? d->num_kv_heads : d->num_heads;         // 0: multi-head attention
    if (kv_heads < 1 || kv_heads > d->num_heads || d->num_heads % kv_heads)
        return exl_set_err(EXL_ERR_ARG, "decode_plan: num_kv_heads (%d) must divide num_heads (%d)", kv_heads, d->num_heads);
    if (kv_heads != d->num_heads && d->tp_world > 1)
        return exl_set_err(EXL_ERR_ARG, "decode_plan: grouped-query attention (%d heads over %d KV heads) under tensor parallelism is not supported by the fused step: use the per-op path", d->num_heads, kv_heads);
    const int HKV = kv_heads * TILE;
    if (H % 512 || HQ % TILE || I % TILE) return exl_set_err(EXL_ERR_ARG, "decode_plan: widths must be multiples of 128 (hidden of 512): hidden %d attn %d inter %d", H, HQ, I);
    const int gs = q0->groupsize;
    int gs32 = gs / 32, sh = 0;
    if (q0->groups > 1) {
        if (gs % 32 || (gs32 & (gs32 - 1))) return exl_set_err(EXL_ERR_ARG, "decode_plan: groupsize %d must be 32 * 2^n", gs);
        while ((1 << sh) < gs32) sh++;
    } else sh = 30;
    std::vector<LayerDesc> L((size_t)d->n_layers);
    bool any_act = false;
    const int expectK[7] = {H, H, H, HQ, H, H, I}, expectN[7] = {HQ, HKV, HKV, H, I, I, H};      // k, v: kv_heads * 128 wide
    for (int l = 0; l < d->n_layers; l++) {
        memset(&L[l], 0, sizeof(LayerDesc));
        for (int i = 0; i < 7; i++) {
            const exl_q4_matrix* w = d->mats[l * 7 + i];
            if (!w) return exl_set_err(EXL_ERR_STATE, "decode_plan: NULL handle (layer %d matrix %d)", l, i);
            if (w->x_map) any_act = true;
            if (w->K != expectK[i] || w->N != expectN[i] || w->device != q0->device)
                return exl_set_err(EXL_ERR_ARG, "decode_plan: layer %d matrix %d is %d x %d, expected %d x %d", l, i, w->K, w->N, expectK[i], expectN[i]);
            const bool one = q0->groups == 1;
            if ((one && w->groups != 1) || (!one && w->groupsize != gs)) return exl_set_err(EXL_ERR_ARG, "decode_plan: mixed group sizes");
            if (!w->valid3) return exl_set_err(EXL_ERR_ARG, "decode_plan: layer %d matrix %d has no unit tensor maps (width %% 128 != 0)", l, i);
            L[l].tw[i] = w->tmap_w3; L[l].ts[i] = w->tmap_sc; L[l].tz[i] = w->tmap_qz; L[l].xmap[i] = w->x_map;
        }
        L[l].ln1 = (const half*)d->ln1[l]; L[l].ln2 = (const half*)d->ln2[l];
        L[l].kc = (half*)d->key_cache[l]; L[l].vc = (half*)d->value_cache[l];
    }
    exl_decode_plan* p = new exl_decode_plan();
    p->device = q0->device;
    StepArgs& a = p->args;
    memset(&a, 0, sizeof(a));
    a.n_layers = d->n_layers; a.H = H; a.HQ = HQ; a.HKV = HKV; a.I = I; a.heads = d->num_heads; a.max_seq = d->max_seq_len; a.gshift = sh;
    a.kv_heads = kv_heads; a.n_rep = d->num_heads / kv_heads;
    a.eps = d->rms_eps; a.sin = (const half*)d->sin; a.cos = (const half*)d->cos;
    a.final_norm = (const half*)d->final_norm; a.lm_head = (const half*)d->lm_head; a.vocab = d->lm_head ? d->vocab : 0;
    if (d->lm_head && (!d->final_norm || d->vocab % 4)) return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan: lm_head needs final_norm and vocab %% 4 == 0"));
    a.spt_max = spt_max_for(H, HQ, I);
    a.act = any_act ? 1 : 0;
    if (any_act && d->tp_world > 1)
        return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan: act-order matrices under tensor parallelism are not supported by the fused step (o_proj needs the all-gathered attention output): use the per-op path"));
    if (multi && any_act)
        return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan_multi: act-order matrices are not supported by the multi-token step: use exl_decode_plan_create (one token per step) or prefill"));
    if (max_batch > 1 && !multi && (any_act || d->tp_world > 1))
        return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan: a batch (max_batch %d) with %s is not supported by the fused step: use max_batch 1 or the per-op path",
                                        max_batch, any_act ? "act-order matrices" : "tensor parallelism"));
    int dev_smem = 0;
    cudaDeviceGetAttribute(&dev_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, p->device);
    p->grid = ds->num_sms;
    if (const char* eg = getenv("EXL_DS_GRID")) { int v = atoi(eg); if (v >= 1 && v <= ds->num_sms) p->grid = v; }
    // ATT keeps two head segments per CTA: every head needs a CTA of its own in the plan's grid (EXL_DS_GRID included)
    if (d->num_heads > p->grid || d->num_heads > DS_MAX_HEADS)
        return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan: more heads (%d) than the grid's %d CTAs (or than %d)", d->num_heads, p->grid, DS_MAX_HEADS));
    p->max_batch = max_batch;
    p->max_tokens = max_tokens; p->cache_seqs = cache_seqs;
    a.bsz = 1;
    if (multi) {
        const int fits = max_tokens_for(H, HQ, I, d->num_heads, kv_heads, (size_t)dev_smem, p->grid);
        if (max_tokens > fits)
            return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan_multi: max_tokens %d does not fit this model on this GPU (shared memory for %d query vectors per KV head, or more KV heads than %d CTAs): the largest is %d",
                                            max_tokens, max_tokens * a.n_rep, p->grid, fits));
        a.xst = batch_xstages(H, HQ, HKV, I, p->grid);
    } else if (max_batch > 1) {
        const int fits = max_batch_for(H, HQ, I, d->num_heads, kv_heads, false, (size_t)dev_smem, p->grid);
        if (max_batch > fits)
            return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan: max_batch %d does not fit this model on this GPU (shared memory, or more virtual heads than %d CTAs): the largest batch is %d",
                                            max_batch, p->grid, fits));
        a.xst = batch_xstages(H, HQ, HKV, I, p->grid);
    }
    const size_t fixed = multi ? smem_fixed_bytes_multi(H, a.n_rep, max_tokens, a.xst) : smem_fixed_bytes(H, HQ, I, any_act, a.n_rep, max_batch, a.xst);
    int depth = ring_depth_for((size_t)dev_smem, fixed);
    if (const char* e = getenv("EXL_DS_DEPTH")) { int v = atoi(e); if (v >= 1 && v < depth) depth = v; }
    if (depth < 2) return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan: model too wide for the shared-memory plan (%d ring stages per pipeline)", depth));
    a.depth = depth;
    p->smem = smem_dynamic_bytes(fixed, depth);
    if ((size_t)H * 2 > (size_t)a.spt_max * 256) return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan: internal: head staging does not fit"));
    const void* kfn = multi ? multi_kernel() : step_kernel_for(any_act, d->tp_world > 1, a.n_rep > 1, max_batch > 1, lora != nullptr);
    // the attribute belongs to the kernel, not the plan: it only grows, so that plans of one kernel with different shared memory
    // (a speculative target and its draft) can be stepped in any order
    cudaFuncAttributes fa{};
    cudaError_t e = cudaFuncGetAttributes(&fa, kfn);
    if (e == cudaSuccess && (size_t)fa.maxDynamicSharedSizeBytes < p->smem)
        e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem);
    if (e != cudaSuccess) return plan_fail(p, exl_set_err(EXL_ERR_CUDA, "decode_plan: smem attribute (%zu B): %s", p->smem, cudaGetErrorString(e)));
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kfn, DS_THREADS, p->smem);
    if (e != cudaSuccess || per_sm < 1) return plan_fail(p, exl_set_err(EXL_ERR_CUDA, "decode_plan: kernel does not fit an SM (smem %zu)", p->smem));
    a.att_slots = multi ? att_slots_multi(p->grid, kv_heads) : att_slots_for(p->grid, d->num_heads, kv_heads);      // the most CTAs per head: one sequence
    // scratch: accumulators | attention partials | barrier (accumulators and partials: max_batch rows / virtual heads)
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
    const size_t mb = (size_t)max_batch;
    const size_t o_qkv = take(mb * (HQ + 2 * HKV) * 4), o_o = take(mb * H * 4), o_gu = take(mb * 2 * I * 4), o_d = take(mb * H * 4);
    const size_t o_att = take(mb * d->num_heads * a.att_slots * PART_LD * 4), o_bar = take(256), o_av = take((size_t)HQ * 2);
    const bool want_trace = getenv("EXL_DS_TRACE") != nullptr;
    const size_t o_trace = want_trace ? take((size_t)p->grid * TRACE_LAYERS * 24 * 8) : 0;
    // LoRA: t accumulators, [max_batch][rank] per adapted matrix
    std::vector<LoraMat> lm(lora ? (size_t)d->n_layers * 7 : 0);
    size_t t_floats = 0;
    for (size_t i = 0; i < lm.size(); i++) {
        lm[i].rank = lora->rank[i];
        lm[i].a = lm[i].rank ? (const half*)lora->a[i] : nullptr; lm[i].b = lm[i].rank ? (const half*)lora->b[i] : nullptr;
        lm[i].t_off = (int)t_floats;
        t_floats += mb * (size_t)lm[i].rank;
    }
    const size_t o_lt = lora ? take(t_floats * 4) : 0;
    const int W = d->tp_world > 1 ? d->tp_world : 1;
    p->shared_o = 0; p->shared_d = (((size_t)W * H * 8) + 255) & ~(size_t)255; p->shared_bar = 2 * p->shared_d;
    const size_t shared_bytes = p->shared_bar + 256;
    if (cudaMalloc(&p->d_scratch, off) != cudaSuccess || cudaMalloc(&p->d_layers, sizeof(LayerDesc) * L.size()) != cudaSuccess ||
        cudaMalloc(&p->d_shared, shared_bytes) != cudaSuccess)
        return plan_fail(p, exl_set_err(EXL_ERR_CUDA, "decode_plan: cudaMalloc failed"));
    if (cudaMemset(p->d_scratch, 0, off) != cudaSuccess || cudaMemset(p->d_shared, 0, shared_bytes) != cudaSuccess ||
        cudaMemcpy(p->d_layers, L.data(), sizeof(LayerDesc) * L.size(), cudaMemcpyHostToDevice) != cudaSuccess)
        return plan_fail(p, exl_set_err(EXL_ERR_CUDA, "decode_plan: upload failed"));
    a.layers = p->d_layers;
    a.acc_qkv = (float*)(p->d_scratch + o_qkv); a.acc_gu = (float*)(p->d_scratch + o_gu);
    a.acc_o = (float*)(p->d_scratch + o_o); a.acc_d = (float*)(p->d_scratch + o_d);
    a.slots_o = (const uint2*)(p->d_shared + p->shared_o); a.slots_d = (const uint2*)(p->d_shared + p->shared_d);
    a.launch_ctr = (unsigned*)(p->d_scratch + o_bar + 64);
    a.attn_vec = (half*)(p->d_scratch + o_av);
    a.tp_rank = d->tp_world > 1 ? d->tp_rank : 0; a.tp_world = d->tp_world > 1 ? d->tp_world : 1;
    if (a.tp_world > 8 || a.tp_rank < 0 || a.tp_rank >= a.tp_world) return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan: bad tensor-parallel rank %d / world %d", d->tp_rank, d->tp_world));
    a.tp_reduce = a.tp_world >= 4 ? 1 : 0;
    if (const char* er = getenv("EXL_DS_TP_REDUCE")) a.tp_reduce = (atoi(er) != 0 && a.tp_world > 1) ? 1 : 0;
    p->peer_base[a.tp_rank] = p->d_shared;
    a.push_o[a.tp_rank] = nullptr; a.push_d[a.tp_rank] = nullptr;
    p->peers_ready = a.tp_world == 1;
    a.att_part = (float*)(p->d_scratch + o_att); a.bar = (unsigned long long*)(p->d_scratch + o_bar);
    if (const char* ed = getenv("EXL_DS_DEBUG")) a.debug = atoi(ed);
    a.trace = want_trace ? (unsigned long long*)(p->d_scratch + o_trace) : nullptr;
    if (lora) {
        static_assert(MAX_BATCH * (TILE + LORA_MAX_RANK) <= LORA_SCRATCH_ROOM, "LA scratch (lora_scratch_floats) exceeds the attention partial area");
        if (cudaMalloc(&p->d_lora, sizeof(LoraMat) * lm.size()) != cudaSuccess ||
            cudaMemcpy(p->d_lora, lm.data(), sizeof(LoraMat) * lm.size(), cudaMemcpyHostToDevice) != cudaSuccess)
            return plan_fail(p, exl_set_err(EXL_ERR_CUDA, "decode_plan: LoRA table upload failed"));
        a.lora = p->d_lora; a.lora_t = (float*)(p->d_scratch + o_lt); a.lora_t4 = (int)(t_floats / 4);
        p->lora_barriers = lora_barriers(lora->rank, d->n_layers);
    }
    *out = p;
    return EXL_OK;
}

extern "C" int exl_decode_plan_destroy(exl_decode_plan* p)
{
    if (!p) return EXL_OK;
    DeviceGuard guard(p->device);
    cudaDeviceSynchronize();
    plan_fail(p, 0);
    return EXL_OK;
}

// Tensor parallel: the region peers reduce into is exported as a cudaIpc handle (64 bytes) ...
extern "C" int exl_decode_plan_ipc_export(exl_decode_plan* p, void* handle64)
{
    if (!p || !handle64) return exl_set_err(EXL_ERR_STATE, "decode_plan_ipc_export: NULL argument");
    DeviceGuard guard(p->device);
    cudaIpcMemHandle_t h;
    EXL_CUDA_TRY(cudaIpcGetMemHandle(&h, p->d_shared));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle size");
    memcpy(handle64, &h, 64);
    return EXL_OK;
}

// ... and every rank imports all ranks' handles (world x 64 bytes, in rank order; its own entry is ignored) before the first step.
extern "C" int exl_decode_plan_ipc_import(exl_decode_plan* p, const void* handles, int world)
{
    if (!p || !handles) return exl_set_err(EXL_ERR_STATE, "decode_plan_ipc_import: NULL argument");
    if (world != p->args.tp_world) return exl_set_err(EXL_ERR_ARG, "decode_plan_ipc_import: %d handles for a world of %d", world, p->args.tp_world);
    DeviceGuard guard(p->device);
    StepArgs& a = p->args;
    for (int r = 0; r < world; r++) {
        if (r == a.tp_rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, (const unsigned char*)handles + (size_t)r * 64, 64);
        void* base = nullptr;
        EXL_CUDA_TRY(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
        p->peer_base[r] = (unsigned char*)base;
        a.push_o[r] = (uint2*)(p->peer_base[r] + p->shared_o) + (size_t)a.tp_rank * a.H;
        a.push_d[r] = (uint2*)(p->peer_base[r] + p->shared_d) + (size_t)a.tp_rank * a.H;
    }
    p->peers_ready = true;
    return EXL_OK;
}

extern "C" int exl_decode_plan_info(const exl_decode_plan* p, int* grid, int* ring_stages, int64_t* smem_bytes, int64_t* barriers_per_step)
{
    if (!p) return exl_set_err(EXL_ERR_STATE, "decode_plan_info: NULL plan");
    if (grid) *grid = p->grid; if (ring_stages) *ring_stages = 4 * p->args.depth; if (smem_bytes) *smem_bytes = (int64_t)p->smem;
    if (barriers_per_step) *barriers_per_step = 1 + (5 + (p->args.act ? 1 : 0) + (p->args.tp_world > 1 ? (p->args.tp_reduce ? 4 : 2) : 0)) * (int64_t)p->args.n_layers
                                                           + p->lora_barriers;
    return EXL_OK;
}

// EXL_DS_TRACE=1 at plan creation: copies the [grid][4 layers][16 events] globaltimer stamps of the last launch to the host
extern "C" int exl_decode_plan_trace(exl_decode_plan* p, unsigned long long* out_host, int64_t capacity)
{
    if (!p || !p->args.trace) return exl_set_err(EXL_ERR_STATE, "decode_plan_trace: plan has no trace buffer (set EXL_DS_TRACE=1 before creating it)");
    const int64_t n = (int64_t)p->grid * TRACE_LAYERS * 24;
    if (capacity < n) return exl_set_err(EXL_ERR_ARG, "decode_plan_trace: need room for %lld values", (long long)n);
    DeviceGuard guard(p->device);
    EXL_CUDA_TRY(cudaMemcpy(out_host, p->args.trace, (size_t)n * 8, cudaMemcpyDeviceToHost));
    return EXL_OK;
}

// the table reset (when `reset`) and the cooperative launch of kernel `kfn` with arguments `a`
static int launch_step(exl_decode_plan* p, StepArgs& a, const void* kfn, bool reset, void* stream_)
{
    if (reset) {
        // short context: some CTAs inside a head's CTA range own no attention unit in this launch (stateless test, so a captured
        // CUDA graph -- past_len is baked into it -- replays the same decision)
        const int n = a.bsz * a.heads * a.att_slots * PART_LD;
        att_part_reset_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream_>>>(a.att_part, n);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        cudaError_t er = cudaGetLastError();
        if (er != cudaSuccess) return exl_set_err(EXL_ERR_CUDA, "launch of att_part_reset_kernel failed: %s", cudaGetErrorString(er));
    }
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeCooperative; at[0].val.cooperative = 1;      // all CTAs co-resident: the grid barrier relies on it
    cfg.gridDim = dim3((unsigned)p->grid); cfg.blockDim = dim3(DS_THREADS); cfg.dynamicSmemBytes = p->smem; cfg.stream = (cudaStream_t)stream_;
    cfg.attrs = at; cfg.numAttrs = 1;
    void* kargs[1] = {(void*)&a};
    cudaError_t e = cudaLaunchKernelExC(&cfg, kfn, kargs);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    if (e != cudaSuccess) return exl_set_err(EXL_ERR_CUDA, "launch of decode_step_kernel failed: %s (grid %d, smem %zu)", cudaGetErrorString(e), p->grid, p->smem);
    return EXL_OK;
}

static int reject_multi_plan(const exl_decode_plan* p)
{
    return exl_set_err(EXL_ERR_ARG, "decode_step: this plan carries up to %d tokens of one sequence per step: call exl_decode_step_multi "
                                    "(or create the plan with exl_decode_plan_create / exl_decode_plan_create_batch)", p->max_tokens);
}

extern "C" int exl_decode_step(exl_decode_plan* p, const void* x_in, int past_len, void* x_out, void* logits, void* stream_)
{
    if (!p) return exl_set_err(EXL_ERR_STATE, "decode_step: NULL plan");
    if (p->max_tokens) return reject_multi_plan(p);
    if (past_len < 0 || past_len >= p->args.max_seq) return exl_set_err(EXL_ERR_ARG, "decode_step: past_len %d outside the cache (max_seq %d)", past_len, p->args.max_seq);
    return exl_decode_step_batch(p, x_in, 1, &past_len, x_out, logits, stream_);
}

extern "C" int exl_decode_step_batch(exl_decode_plan* p, const void* x_in, int bsz, const int* past_len_host, void* x_out, void* logits, void* stream_)
{
    if (!p) return exl_set_err(EXL_ERR_STATE, "decode_step: NULL plan");
    if (p->max_tokens) return reject_multi_plan(p);
    if (!x_in) return exl_set_err(EXL_ERR_ARG, "decode_step: x_in is NULL");
    if (bsz < 1 || bsz > p->max_batch)
        return exl_set_err(EXL_ERR_ARG, "decode_step: bsz %d outside 1..%d (the plan's max_batch): create the plan with exl_decode_plan_create_batch for a larger batch", bsz, p->max_batch);
    if (!past_len_host) return exl_set_err(EXL_ERR_ARG, "decode_step: past_len is NULL");
    int longest = 0;
    for (int b = 0; b < bsz; b++) {
        if (past_len_host[b] < 0 || past_len_host[b] >= p->args.max_seq)
            return exl_set_err(EXL_ERR_ARG, "decode_step: past_len[%d] = %d outside the cache (max_seq %d)", b, past_len_host[b], p->args.max_seq);
        longest = past_len_host[b] > longest ? past_len_host[b] : longest;
    }
    if (p->args.lm_head && !logits) return exl_set_err(EXL_ERR_ARG, "decode_step: the plan has an lm_head, logits must be given");
    if (!p->peers_ready) return exl_set_err(EXL_ERR_STATE, "decode_step: tensor-parallel plan: call exl_decode_plan_ipc_import first");
    DeviceGuard guard(p->device);
    StepArgs a = p->args;
    a.x_in = (const half*)x_in; a.x_out = (half*)x_out; a.logits = (float*)logits; a.past_len = longest;
    a.bsz = bsz;
    for (int b = 0; b < bsz; b++) a.past_lens[b] = past_len_host[b];
    return launch_step(p, a, step_kernel_for(a.act != 0, a.tp_world > 1, a.n_rep > 1, p->max_batch > 1, a.lora != nullptr),
                       att_needs_reset(a.heads, a.kv_heads, longest, p->grid, bsz), stream_);
}

extern "C" int exl_decode_step_multi(exl_decode_plan* p, const void* x_in, int n, int seq, int past_len, void* x_out, void* logits, void* stream_)
{
    if (!p) return exl_set_err(EXL_ERR_STATE, "decode_step_multi: NULL plan");
    if (!p->max_tokens)
        return exl_set_err(EXL_ERR_ARG, "decode_step_multi: the plan is not a multi-token plan: create it with exl_decode_plan_create_multi, "
                                        "or step it with exl_decode_step / exl_decode_step_batch");
    if (!x_in) return exl_set_err(EXL_ERR_ARG, "decode_step_multi: x_in is NULL");
    if (n < 1 || n > p->max_tokens)
        return exl_set_err(EXL_ERR_ARG, "decode_step_multi: n %d outside 1..%d (the plan's max_tokens): split the chunk, or create the plan with a larger max_tokens", n, p->max_tokens);
    if (seq < 0 || seq >= p->cache_seqs)
        return exl_set_err(EXL_ERR_ARG, "decode_step_multi: seq %d outside the caches' sequences [0, %d)", seq, p->cache_seqs);
    if (past_len < 0 || past_len + n > p->args.max_seq)
        return exl_set_err(EXL_ERR_ARG, "decode_step_multi: past_len %d + n %d outside the cache (max_seq %d): rows [%d, %d) must fit", past_len, n, p->args.max_seq, past_len, past_len + n);
    if (p->args.lm_head && !logits) return exl_set_err(EXL_ERR_ARG, "decode_step_multi: the plan has an lm_head, logits must be given");
    DeviceGuard guard(p->device);
    StepArgs a = p->args;
    a.x_in = (const half*)x_in; a.x_out = (half*)x_out; a.logits = (float*)logits; a.past_len = past_len;
    a.bsz = n; a.seq = seq;
    for (int b = 0; b < n; b++) a.past_lens[b] = past_len;
    return launch_step(p, a, multi_kernel(), att_needs_reset_multi(a.heads, a.kv_heads, past_len, p->grid), stream_);
}
