// decode_step.cu -- ONE persistent cooperative kernel for a whole decode token (bsz 1, q_len 1) on sm_90a.
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
//    NEXT phase is already in flight while the consumers are in a barrier or in a phase prologue.  HBM stays busy across
//    phase and layer boundaries -- the thing separate launches could not do.
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
//  * ATT: (head, 16-position chunk) units, online softmax per warp in fp32 (as decode_attn.cu), partial (m, l, o) per CTA to
//    L2, combined in the O prologue.  The newest K/V row never round-trips through HBM before it is used.
//  * HEAD: lm_head [vocab, hidden] fp16 streamed as 8 KB stages, fp32 dot products, fp32 logits by red.global.add.
//
// Restrictions (checked on the host; anything else uses the per-op kernels): head_dim 128, kv_heads == heads, groupsize 32 * 2^n
// (or one group), widths multiples of 128, act-order only without tensor parallelism (template flag ACT: x is gathered through
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
constexpr int DS_MAX_HEADS = 256;                // (local) heads a plan may have: size of the per-head CTA-range table
enum { ZR_QKV = 0, ZR_H = 1, ZR_GU = 2, ZR_LOGITS = 3, ZR_HALF = 4, ZR_COUNT = 5 };     // zero_share / push ranges
constexpr unsigned long long WAIT_NS = 4000000000ull;   // any single wait longer than this aborts the launch

struct alignas(64) LayerDesc
{
    CUtensorMap tw[7];                 // q k v o gate up down: exl_q4_matrix::tmap_w3 (one 8 KB unit per op)
    CUtensorMap ts[7];                 // ::tmap_sc
    CUtensorMap tz[7];                 // ::tmap_qz
    const uint32_t* xmap[7];           // act-order: x column feeding sequential row k of each matrix (exl_q4_matrix::x_map), else NULL
    const half* ln1; const half* ln2;
    half* kc; half* vc;                // [heads, max_seq, 128]
};

struct StepArgs
{
    const LayerDesc* layers; int n_layers;
    int H, HQ, I;                      // hidden, attention width (heads * 128), intermediate width
    int heads, max_seq, past_len;
    int gshift;                        // log2(groupsize / 32); 30 = one group per matrix
    int depth;                         // ring stages per pipeline (4 pipelines)
    int spt_max;                       // max K / 128 over the phases
    int act;                           // act-order matrices present: x is gathered through each matrix's x_map while it is staged; the
                                       // matrices of a phase then need their own quantised x (two staging slots), and o_proj's input
                                       // (a gather over all heads) goes through one extra combine step + barrier
    half* attn_vec;                    // [HQ] combined attention output (act-order only)
    float eps;
    const half* x_in; half* x_out;     // [H] input hidden state; final hidden state (before the final norm), optional
    const half* sin; const half* cos;  // [max_seq, 128]
    const half* final_norm; const half* lm_head; float* logits; int vocab;     // optional head
    float* acc_qkv; float* acc_o; float* acc_gu; float* acc_d;                 // fp32 phase accumulators in L2
    float* att_part; int att_slots;    // [heads][att_slots][PART_LD]
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
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tmap, int c0, int c1, uint32_t bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 :: "r"(dst), "l"(tmap), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tmap, int c0, int c1, int c2, uint32_t bar)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 :: "r"(dst), "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(bar) : "memory");
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
__device__ __forceinline__ void grid_barrier(unsigned long long* ctr, unsigned long long& target, unsigned nctas, int tid)
{
    consumer_sync();
    if (tid == 0) {
        asm volatile("red.release.gpu.global.add.u64 [%0], 1;" :: "l"(ctr) : "memory");
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

// ACT: act-order matrices present; TP: tensor parallel.  Compile-time so that the common kernel (neither) carries none of their
// address arithmetic, branches or code (the runtime-flag version of the same source was 10 % slower on the plain 7B step).
template <bool ACT, bool TP>
__global__ void __launch_bounds__(DS_THREADS, 1) decode_step_kernel(const __grid_constant__ StepArgs a)
{
    extern __shared__ __align__(128) unsigned char smem[];
    const int depth = a.depth, nst = 4 * a.depth;
    unsigned char* ring = smem + ((1024u - (smem_u32(smem) & 1023u)) & 1023u);      // nst x STAGE_STRIDE: pipeline g owns stages [g * depth, (g + 1) * depth)
    // staging slot 0: spt_max K stages; act-order adds slot 1 (H / 128 stages: only the multi-matrix phases, whose K is H, need it --
    // the two matrices a CTA's range can touch have different x_maps)
    const int xstages = a.spt_max + (ACT ? a.H / TILE : 0);
    const uint32_t xs_slot = (uint32_t)a.spt_max * 256u, seg_slot = (uint32_t)a.spt_max * 32u;
    unsigned char* xs = ring + (size_t)nst * STAGE_STRIDE;                            // xstages x 16 k8-rows x 16 B: quantised x planes by K stage
    unsigned char* segt = xs + (size_t)xstages * 256;                                  // xstages x 4 x {sum x_q, x scale}
    half* xres = reinterpret_cast<half*>(segt + (size_t)xstages * 32);                // [H] residual stream (fp16, as the reference keeps it)
    float* parts = reinterpret_cast<float*>(xres + a.H);                               // [2 segments][17][PART_LD] attention partials of the warps (+ the new token)
    float* q_s = parts + 2 * 17 * PART_LD;                                             // [2][128] scaled q of the segment's head
    float* kn_s = q_s + 2 * TILE;                                                      // [2][128] newest k row (after rope)
    float* vn_s = kn_s + 2 * TILE;                                                     // [2][128] newest v row
    half* qh_s = reinterpret_cast<half*>(vn_s + 2 * TILE);                             // [2][128] q of the segment's head after rope, fp16 as the reference holds it (unscaled)
    unsigned char* wnorm = reinterpret_cast<unsigned char*>(qh_s + 2 * TILE);          // [H / 8][16 B]: norm weights of the rows this CTA quantises next (by k8-row slot)
    half* xh = reinterpret_cast<half*>(xs);                                            // HEAD: normalised x [H] (xs is free by then)
    __shared__ __align__(8) unsigned long long full_bar[4 * MAX_DEPTH], empty_bar[4 * MAX_DEPTH];
    __shared__ float s_red[DS_NCW];
    __shared__ unsigned long long s_base, s_base_x;
    // The schedule does not depend on the layer (nor, except ATT, on anything but the shapes): this CTA's unit range of every phase,
    // its shares of the buffers it zeroes and the CTA range of every head's attention units are computed ONCE per launch.  (They were
    // 64-bit divisions re-done by every thread in every phase of every layer: 5 % of all instructions executed, in the prologues.)
    __shared__ int s_rng[6][4];                                  // [phase kind]{lo, hi, first K stage lo % spt, K stages to quantise min(hi - lo, spt)}
    __shared__ int s_zr[ZR_COUNT][2];                            // [buffer][lo, hi) in units of 4 floats (ZR_HALF: 2 floats)
    __shared__ unsigned short s_clo[DS_MAX_HEADS], s_chi[DS_MAX_HEADS];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int G = (int)gridDim.x, cta = (int)blockIdx.x;

    if (tid == 0) {
        for (int i = 0; i < nst; i++) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (tid >= 32 && tid < 38) {
        const Phase p = phase_of(a, tid - 32, G);
        const int lo = range_lo(p.U, cta, p.G), hi = range_lo(p.U, cta + 1, p.G);
        s_rng[tid - 32][0] = lo; s_rng[tid - 32][1] = hi;
        s_rng[tid - 32][2] = (p.spt > 0 && hi > lo) ? lo % p.spt : 0;
        s_rng[tid - 32][3] = p.spt > 0 ? min(hi - lo, p.spt) : 0;
    } else if (tid >= 64 && tid < 64 + ZR_COUNT) {
        const int k = tid - 64;
        const int n = k == ZR_QKV ? (3 * a.HQ) >> 2 : (k == ZR_H ? a.H >> 2 : (k == ZR_GU ? (2 * a.I) >> 2 : (k == ZR_LOGITS ? a.vocab >> 2 : a.H >> 1)));
        s_zr[k][0] = share_lo(n, cta, G); s_zr[k][1] = share_lo(n, cta + 1, G);
    } else if (tid >= 128 && tid < 128 + a.heads) {
        const Phase pa = phase_of(a, PH_ATT, G);
        const int h = tid - 128;
        s_clo[h] = (unsigned short)cta_of((long long)h * pa.tpm, pa.U, pa.G);
        s_chi[h] = (unsigned short)cta_of((long long)(h + 1) * pa.tpm - 1, pa.U, pa.G);
    }
    __syncthreads();

    if (warp >= DS_NCW) {
        // ==================== producer warp of pipeline pq: every 4th stage of the token's HBM stream, in schedule order ====================
        const int pq = warp - DS_NCW;
        int ls = 0; uint32_t par = 0; int issued = 0;                       // ls: stage inside the pipeline's ring; par: parity of the empty completion to wait for
        const uint32_t ring_a = smem_u32(ring) + (uint32_t)pq * depth * STAGE_STRIDE;
        const uint32_t full0 = smem_u32(&full_bar[pq * depth]), empty0 = smem_u32(&empty_bar[pq * depth]);
        int jbase = 0;
        auto acquire = [&](uint32_t tx) -> uint32_t {
            if (issued >= depth) mbar_wait(empty0 + ls * 8, par ^ 1u);
            if (lane == 0) mbar_expect_tx(full0 + ls * 8, tx);
            __syncwarp();
            return ring_a + (uint32_t)ls * STAGE_STRIDE;
        };
        auto advance = [&]() { if (issued < depth) issued++; if (++ls == depth) { ls = 0; par ^= 1u; } };
        const int ngrow = a.gshift >= 2 ? 1 : (4 >> a.gshift);          // group rows per K stage (groupsize 32: 4, 64: 2, >= 128: 1)
        #pragma unroll 1
        for (int l = 0; l < a.n_layers; l++) {
            const LayerDesc* L = a.layers + l;
            #pragma unroll 1
            for (int ph = PH_QKV; ph <= PH_DOWN; ph++) {
                const Phase p = phase_of(a, ph, G);
                const int u0 = s_rng[ph][0], u1 = s_rng[ph][1];
                const int i0 = ((pq - jbase) & 3);
                jbase += u1 - u0;
                if (ph == PH_ATT) {
                    int h = (u0 + i0) / p.tpm, ch = (u0 + i0) - h * p.tpm;
                    #pragma unroll 1
                    for (int u = u0 + i0; u < u1; u += 4) {
                        const int pos0 = ch * 16;
                        int nv = a.past_len - pos0; nv = nv < 0 ? 0 : (nv > 16 ? 16 : nv);
                        const uint32_t base = acquire((uint32_t)nv * 512u);
                        if (nv > 0) {
                            const size_t off = ((size_t)h * a.max_seq + pos0) * TILE;
                            if (lane == 0) bulk_g2s(base, L->kc + off, (uint32_t)nv * 256u, full0 + ls * 8);
                            if (lane == 1) bulk_g2s(base + 4096, L->vc + off, (uint32_t)nv * 256u, full0 + ls * 8);
                        }
                        advance();
                        ch += 4;
                        while (ch >= p.tpm) { ch -= p.tpm; h++; }
                    }
                    continue;
                }
                if (u0 + i0 >= u1) continue;
                int tile = (u0 + i0) / p.spt, s = (u0 + i0) - tile * p.spt;
                int mi = tile / p.tpm, ct = tile - mi * p.tpm;
                #pragma unroll 1
                for (int u = u0 + i0; u < u1; u += 4) {
                    const int m = p.mat0 + mi;
                    const uint32_t base = acquire((uint32_t)W_BYTES + (uint32_t)ngrow * 320u);
                    const uint32_t fb = full0 + ls * 8;
                    const int grow = a.gshift >= 2 ? ((s * 4) >> a.gshift) : s * ngrow;
                    if (lane == 0) tma_load_3d(base, &L->tw[m], 0, s * 16, ct * 4, fb);
                    else if (lane == 1) tma_load_2d(base + META_SC, &L->ts[m], ct * TILE, grow, fb);
                    else if (lane == 2) tma_load_2d(base + META_ZQ, &L->tz[m], ct * 16, grow, fb);
                    advance();
                    s += 4;
                    while (s >= p.spt) { s -= p.spt; if (++ct == p.tpm) { ct = 0; mi++; } }
                }
            }
        }
        {
            const int u0 = s_rng[PH_HEAD][0], u1 = s_rng[PH_HEAD][1];
            const int i0 = ((pq - jbase) & 3);
            const long long total = (long long)a.vocab * a.H * 2;
            const unsigned char* src = reinterpret_cast<const unsigned char*>(a.lm_head);
            #pragma unroll 1
            for (int u = u0 + i0; u < u1; u += 4) {
                const long long off = (long long)u * W_BYTES;
                const uint32_t bytes = (uint32_t)((total - off) < W_BYTES ? (total - off) : W_BYTES);
                const uint32_t base = acquire(bytes);
                if (lane == 0) bulk_g2s(base, src + off, bytes, full0 + ls * 8);
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
    for (int i = tid; i < a.H / 8; i += DS_CONSUMERS)
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
    preload_norm(a.layers[0].ln1, phase_of(a, PH_QKV, G));
    grid_barrier(a.bar, target, (unsigned)G, tid);
    if (TP && cta == 0 && tid == 0) *a.launch_ctr = (unsigned)s_base_x + 1u;      // every CTA has read it (it is past the barrier)

    // ---- residual add (fp16(x + fp32 delta), the rounding point of q4_matmul's no_zero epilogue) + row factor of the RMS norm ----
    auto residual_and_norm = [&](const float* delta, const uint2* slots = nullptr, unsigned epoch = 0u) -> float {
        asm volatile("cp.async.wait_all;" ::: "memory");
        float ss = 0.f;
        for (int i = tid; i < a.H / 8; i += DS_CONSUMERS) {
            uint4 xv = reinterpret_cast<uint4*>(xres)[i];
            half2* h = reinterpret_cast<half2*>(&xv);
            if (delta) {
                const float4 own0 = ldcg4(delta + i * 8), own1 = ldcg4(delta + i * 8 + 4);
                float4 d0 = own0, d1 = own1;
                if (TP && slots) {
                    // tensor parallel: the sum over ALL ranks' partials in rank order (bitwise identical on every rank); the peers'
                    // partials sit in this rank's slots as {value, epoch} pairs, polled until the epoch of this (layer, phase) shows up
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
                reinterpret_cast<uint4*>(xres)[i] = xv;
            }
            #pragma unroll
            for (int j = 0; j < 4; j++) { const float2 f = __half22float2(h[j]); ss = fmaf(f.x, f.x, ss); ss = fmaf(f.y, f.y, ss); }
        }
        #pragma unroll
        for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        if (lane == 0) s_red[warp] = ss;
        consumer_sync();                                      // also publishes the updated xres
        float tot = 0.f;
        #pragma unroll
        for (int w = 0; w < DS_NCW; w++) tot += s_red[w];     // same order in every thread
        return __half2float(__float2half_rn(rsqrtf(tot / (float)a.H + a.eps)));       // rms_norm.cu:113-116
    };

    // ---- quantise the K stages [s0, s0 + n) (cyclic mod spt) of the phase input into xs / segt; `get(k8, it)` yields 8 fp16 values ----
    // RPGC = k8-rows per quantisation segment at compile time (16: groupsize >= 128, the common case: unrolled shuffles, shifts instead
    // of divisions) or 0 = the run-time value rpg (groupsize 32 / 64)
    auto stage_x = [&](auto rpg_c, int s0, int n, int spt, auto get, int slot) {
        constexpr int RPGC = decltype(rpg_c)::value;
        const int rp = RPGC ? RPGC : rpg;
        unsigned char* xs_w = xs; unsigned char* seg_w = segt;
        if constexpr (ACT) { xs_w += (size_t)slot * xs_slot; seg_w += (size_t)slot * seg_slot; }
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
                *reinterpret_cast<uint4*>(xs_w + (size_t)s * 256 + rr * 16) = q;
                if ((rr & (rp - 1)) == 0)
                    *reinterpret_cast<float2*>(seg_w + (size_t)s * 32 + (rr / rp) * 8) = make_float2(__int_as_float(sum), mx * (1.0f / 32639.0f));
            }
        }
    };
    auto stage_xd = [&](int s0, int n, int spt, auto get, int slot = 0) {
        if (rpg == 16) stage_x(std::integral_constant<int, 16>{}, s0, n, spt, get, slot);
        else stage_x(std::integral_constant<int, 0>{}, s0, n, spt, get, slot);
    };
    auto norm_get = [&](float rm) {
        return [=](int k8, int it) -> uint4 {
            uint4 xv = reinterpret_cast<const uint4*>(xres)[k8];
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
        const int per_mat = p.tpm * p.spt;
        const int mi0 = u0 / per_mat, mi1 = ACT ? (u1 - 1) / per_mat : mi0;
        for (int mi = mi0; mi <= mi1; mi++) {
            const int ua = ACT ? max(u0, mi * per_mat) : u0, ub = ACT ? min(u1, (mi + 1) * per_mat) : u1;
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
        auto flush_tile = [&]() {
            if (t == 0) {
                const int mi = cur_tile / p.tpm, col0 = (cur_tile - mi * p.tpm) * TILE;
                red_add_v4(p.acc + (size_t)mi * p.N + col0 + lane_col, acc[0], acc[1], acc[2], acc[3]);
            }
            acc[0] = acc[1] = acc[2] = acc[3] = 0.f;
        };
        // every address below is a 32-bit shared-memory address built from per-lane constants computed once per phase
        // B column n of the MMA is supplied by the lanes with g == n: 0 = high-byte plane of x, 1 = low-byte plane.  Columns 2..7 only
        // feed D columns 2..7, which live in lanes t >= 1 and are never read -- so those lanes may load anything (they load plane g & 1).
        const uint32_t x_lane = smem_u32(xs) + t * 16 + (g & 1) * 8;
        constexpr uint32_t xstage = 256u, xunit = 64u;
        const uint32_t w_lane = (uint32_t)(wn * BOX_BYTES + t * 128 + ((pg ^ t) << 4));              // k8-rows t, t + 8 (r & 7 == t)
        const uint32_t w_lane4 = w_lane + 512u + ((pg & 4) ? -64 : 64);                              // k8-rows t + 4, t + 12: chunk (pg ^ t) ^ 4
        const uint32_t sc_lane = (uint32_t)(META_SC + lane_col * 2), zq_lane = (uint32_t)(META_ZQ + (lane_col >> 3) * 4);
        const uint32_t zshift = (uint32_t)((lane_col & 4) * 4);
        const uint32_t seg_a = smem_u32(segt);
        // NOTE: everything act-order specific is under `if constexpr`: with plain runtime-constant code in its place ptxas produced a
        // 10 % slower plain kernel (measured by A/B builds on one box: any one of these blocks removed restored the speed)
        [[maybe_unused]] int mi_first = 0;                  // staging slot of a tile = its matrix - the first matrix of the CTA's range
        [[maybe_unused]] uint32_t xoff = 0u, soff = 0u;
        if constexpr (ACT) { mi_first = (u0 / p.spt) / p.tpm; xoff = (uint32_t)(cur_tile / p.tpm - mi_first) * xs_slot; soff = (uint32_t)(cur_tile / p.tpm - mi_first) * seg_slot; }
        bool ready = mbar_try(full0 + ls * 8, par);
        for (; u < u1; u += 4) {
            if (tile != cur_tile) {
                flush_tile(); cur_tile = tile;
                if constexpr (ACT) { const uint32_t sl = (uint32_t)(tile / p.tpm - mi_first); xoff = sl * xs_slot; soff = sl * seg_slot; }
            }
            const uint32_t tok = mbar_wait_tok(full0 + ls * 8, par, ready);
            const int ls_cur = ls;
            if (++ls == depth) { ls = 0; par ^= 1u; }
            // probe the NEXT stage's barrier now: its ~90-cycle answer overlaps this stage's work
            ready = (u + 4 < u1) ? mbar_try(full0 + ls * 8, par) : false;
            float dep = 0.f;
            if (!(a.debug & 1)) {
                const uint32_t sb = ring_a + (uint32_t)ls_cur * STAGE_STRIDE + tok;
                uint32_t xr = x_lane + (uint32_t)s * xstage + tok;
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
                    else sg[e] = lds64(seg_a + (uint32_t)s * 32u + e * 8 + tok);
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

    float rm = 0.f;
    #pragma unroll 1
    for (int l = 0; l < a.n_layers; l++) {
        const LayerDesc* L = a.layers + l;
        // ======================================================== QKV ========================================================
        {
            const Phase p = phase_of(a, PH_QKV, G);
            const int u0 = s_rng[PH_QKV][0], u1 = s_rng[PH_QKV][1];
            stamp(l, 0);
            if (l > 0) zero_share(a.acc_gu, ZR_GU);
            rm = residual_and_norm(l > 0 ? a.acc_d : nullptr, (TP && !a.tp_reduce && l > 0) ? a.slots_d : nullptr, epoch0 + 2u * (l - 1) + 1u);
            stamp(l, 15);
            if constexpr (!ACT) { if (u1 > u0) stage_xd(s_rng[p.kind][2], s_rng[p.kind][3], p.spt, norm_get(rm)); }
            else stage_phase(p, u0, u1, [&](int m) { return norm_get_map(L->ln1, rm, L->xmap[m]); });
            consumer_sync();
            stamp(l, 1);
            gemv(p, u0, u1);
            jbase += u1 - u0;
            stamp(l, 2);
        }
        grid_barrier(a.bar, target, (unsigned)G, tid);
        stamp(l, 3);

        // ======================================================== ATT ========================================================
        {
            const Phase p = phase_of(a, PH_ATT, G);
            const int u0 = s_rng[PH_ATT][0], u1 = s_rng[PH_ATT][1];
            if (l > 0) zero_share(a.acc_d, ZR_H);
            const int nph = p.tpm;
            const float scale = rsqrtf((float)TILE);
            const int l16 = lane & 15, sub = lane >> 4;
            const int h0 = u1 > u0 ? u0 / nph : 0;
            const int nseg = u1 > u0 ? (u1 - 1) / nph - h0 + 1 : 0;            // <= 2 (heads <= grid, checked on the host)
            // every segment's q (and the new k / v rows where this CTA owns the head's last chunk): one L2 round trip
            if (tid < nseg * TILE) {
                const int sg = tid >> 7, d = tid & 127, h = h0 + sg;
                const bool owner = min(u1, (h + 1) * nph) == (h + 1) * nph;
                // fp16 projection result, rope in fp16 with the reference's instruction order (rope.cu:48-67)
                const half* sr = a.sin + (size_t)a.past_len * TILE;
                const half* cr = a.cos + (size_t)a.past_len * TILE;
                const float* aq = a.acc_qkv + (size_t)h * TILE;
                const half qv = __float2half_rn(__ldcg(aq + d)), qo = __float2half_rn(__ldcg(aq + (d ^ 64)));
                const half sn = d < 64 ? __hneg(sr[d]) : sr[d];
                const half qr = __hfma(qv, cr[d], __hmul(qo, sn));
                qh_s[sg * TILE + d] = qr;
                q_s[sg * TILE + d] = __half2float(qr) * scale;
                if (owner) {
                    const float* ak = a.acc_qkv + a.HQ + (size_t)h * TILE;
                    const half kv = __float2half_rn(__ldcg(ak + d)), ko = __float2half_rn(__ldcg(ak + (d ^ 64)));
                    const half kr = __hfma(kv, cr[d], __hmul(ko, sn));
                    const half vv = __float2half_rn(__ldcg(a.acc_qkv + 2 * a.HQ + (size_t)h * TILE + d));
                    kn_s[sg * TILE + d] = __half2float(kr); vn_s[sg * TILE + d] = __half2float(vv);
                    const size_t off = ((size_t)h * a.max_seq + a.past_len) * TILE + d;      // cache layout q4_attn.cu:32-51
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
                    int nv = a.past_len - ch * 16; nv = nv < 0 ? 0 : (nv > 16 ? 16 : nv);
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
            jbase += u1 - u0;
            stamp(l, 4);
        }
        grid_barrier(a.bar, target, (unsigned)G, tid);
        stamp(l, 5);

        // ========================================================= O =========================================================
        {
            const Phase p = phase_of(a, PH_O, G);
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
                // stage k of o_proj is head k: the CTA combines exactly the heads its K range needs
                if (u1 > u0) stage_xd(s_rng[PH_O][2], s_rng[PH_O][3], p.spt, [&](int k8, int) -> uint4 { return combine8(k8 >> 4, (k8 & 15) * 8); });
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
            stamp(l, 6);
            gemv(p, u0, u1);
            jbase += u1 - u0;
            preload_norm(L->ln2, phase_of(a, PH_GU, G));
            stamp(l, 7);
        }
        if constexpr (TP) push_partial(a.acc_o, a.push_o, epoch0 + 2u * l, l, 16);
        else grid_barrier(a.bar, target, (unsigned)G, tid);
        stamp(l, 8);

        // ========================================================= GU ========================================================
        {
            const Phase p = phase_of(a, PH_GU, G);
            const int u0 = s_rng[PH_GU][0], u1 = s_rng[PH_GU][1];
            rm = residual_and_norm(a.acc_o, (TP && !a.tp_reduce) ? a.slots_o : nullptr, epoch0 + 2u * l);
            if constexpr (!ACT) { if (u1 > u0) stage_xd(s_rng[p.kind][2], s_rng[p.kind][3], p.spt, norm_get(rm)); }
            else stage_phase(p, u0, u1, [&](int m) { return norm_get_map(L->ln2, rm, L->xmap[m]); });
            consumer_sync();
            stamp(l, 9);
            gemv(p, u0, u1);
            jbase += u1 - u0;
            stamp(l, 10);
        }
        grid_barrier(a.bar, target, (unsigned)G, tid);
        stamp(l, 11);

        // ======================================================== DOWN =======================================================
        {
            const Phase p = phase_of(a, PH_DOWN, G);
            const int u0 = s_rng[PH_DOWN][0], u1 = s_rng[PH_DOWN][1];
            zero_share(a.acc_o, ZR_H);
            if constexpr (!ACT) {
                if (u1 > u0) stage_xd(s_rng[PH_DOWN][2], s_rng[PH_DOWN][3], p.spt, [&](int k8, int) -> uint4 {
                    // silu(gate) * up on the fp16-rounded projections (q4_mlp.cu:27-36,46-88)
                    const float4 g0 = ldcg4(a.acc_gu + k8 * 8), g1 = ldcg4(a.acc_gu + k8 * 8 + 4);
                    const float4 u0v = ldcg4(a.acc_gu + a.I + k8 * 8), u1v = ldcg4(a.acc_gu + a.I + k8 * 8 + 4);
                    const float gf[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
                    const float uf[8] = {u0v.x, u0v.y, u0v.z, u0v.w, u1v.x, u1v.y, u1v.z, u1v.w};
                    uint4 r; half* hh = reinterpret_cast<half*>(&r);
                    #pragma unroll
                    for (int i = 0; i < 8; i++) hh[i] = __hmul(silu_h(__float2half_rn(gf[i])), __float2half_rn(uf[i]));
                    return r;
                });
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
            stamp(l, 12);
            gemv(p, u0, u1);
            jbase += u1 - u0;
            if (l + 1 < a.n_layers) preload_norm(a.layers[l + 1].ln1, phase_of(a, PH_QKV, G));
            stamp(l, 13);
        }
        if constexpr (TP) push_partial(a.acc_d, a.push_d, epoch0 + 2u * l + 1u, l, 18);
        else grid_barrier(a.bar, target, (unsigned)G, tid);
        stamp(l, 14);
    }

    // ========================================================= HEAD ==========================================================
    rm = residual_and_norm(a.n_layers > 0 ? a.acc_d : nullptr, (TP && !a.tp_reduce && a.n_layers > 0) ? a.slots_d : nullptr, epoch0 + 2u * (a.n_layers - 1) + 1u);
    if (a.x_out && cta == 0)
        for (int i = tid; i < a.H / 8; i += DS_CONSUMERS) reinterpret_cast<uint4*>(a.x_out)[i] = reinterpret_cast<const uint4*>(xres)[i];
    if (a.lm_head) {
        const Phase p = phase_of(a, PH_HEAD, G);
        const int u0 = s_rng[PH_HEAD][0], u1 = s_rng[PH_HEAD][1];
        {
            const half2 rm2 = __float2half2_rn(rm);
            for (int i = tid; i < a.H / 8; i += DS_CONSUMERS) {
                uint4 xv = reinterpret_cast<const uint4*>(xres)[i];
                const uint4 wv = __ldg(reinterpret_cast<const uint4*>(a.final_norm) + i);
                half2* h = reinterpret_cast<half2*>(&xv); const half2* w2 = reinterpret_cast<const half2*>(&wv);
                #pragma unroll
                for (int q = 0; q < 4; q++) h[q] = __hmul2(__hmul2(h[q], rm2), w2[q]);
                reinterpret_cast<uint4*>(xh)[i] = xv;
            }
        }
        consumer_sync();
        // stage = 8 chunks of 512 fp16 of the row-major [vocab, H] matrix; the 4 warps of the pipeline take 2 chunks each
        const int cpr = a.H >> 9;                               // chunks per vocabulary row
        const long long nchunks = (long long)a.vocab * cpr;
        for (int u = u0 + ((wk - jbase) & 3); u < u1; u += 4) {
            mbar_wait(full0 + ls * 8, par);
            const unsigned char* sb = ring + (size_t)(wk * depth + ls) * STAGE_STRIDE;
            const long long c0 = (long long)u * 8 + wn * 2;
            long long row = c0 / cpr; int kc = (int)(c0 - row * cpr);
            float part = 0.f;
            #pragma unroll 1
            for (int cc = 0; cc < ((a.debug & 4) ? 0 : 2) && c0 + cc < nchunks; cc++) {
                #pragma unroll
                for (int hf = 0; hf < 2; hf++) {
                    const uint4 wv = *reinterpret_cast<const uint4*>(sb + (wn * 2 + cc) * 1024 + hf * 512 + lane * 16);
                    const uint4 xv = *reinterpret_cast<const uint4*>(reinterpret_cast<const unsigned char*>(xh) + (size_t)kc * 1024 + hf * 512 + lane * 16);
                    part = fhfma2(wv.x, xv.x, part); part = fhfma2(wv.y, xv.y, part);
                    part = fhfma2(wv.z, xv.z, part); part = fhfma2(wv.w, xv.w, part);
                }
                if (++kc == cpr || cc == 1 || c0 + cc + 1 == nchunks) {
                    float tot = part;
                    #pragma unroll
                    for (int off = 16; off > 0; off >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, off);
                    if (lane == 0) atomicAdd(a.logits + row, tot);
                    part = 0.f;
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
};

static const void* step_kernel_for(bool act, bool tp)
{
    if (act) return tp ? (const void*)decode_step_kernel<true, true> : (const void*)decode_step_kernel<true, false>;
    return tp ? (const void*)decode_step_kernel<false, true> : (const void*)decode_step_kernel<false, false>;
}

static int plan_fail(exl_decode_plan* p, int rc)
{
    if (p) {
        for (int r = 0; r < 8; r++) if (p->peer_base[r] && p->peer_base[r] != p->d_shared) cudaIpcCloseMemHandle(p->peer_base[r]);
        if (p->d_layers) cudaFree(p->d_layers);
        if (p->d_scratch) cudaFree(p->d_scratch);
        if (p->d_shared) cudaFree(p->d_shared);
        delete p;
    }
    return rc;
}

extern "C" int exl_decode_plan_create(const exl_decode_desc* d, exl_decode_plan** out)
{
    if (!d || !out) return exl_set_err(EXL_ERR_ARG, "decode_plan: NULL argument");
    *out = nullptr;
    if (d->n_layers < 1 || d->n_layers > MAX_LAYERS || !d->mats || !d->mats[0]) return exl_set_err(EXL_ERR_ARG, "decode_plan: bad layer count %d", d->n_layers);
    const exl_q4_matrix* q0 = d->mats[0];
    ExlDevice* ds = exl_device_state(q0->device);
    if (!ds) return EXL_ERR_CUDA;
    DeviceGuard guard(q0->device);
    const int H = q0->K, HQ = q0->N, I = d->mats[4]->N;
    if (d->head_dim != TILE || d->num_heads * TILE != HQ) return exl_set_err(EXL_ERR_ARG, "decode_plan: head_dim must be 128 and heads * 128 == q_proj width (%d heads, width %d)", d->num_heads, HQ);
    if (H % 512 || HQ % TILE || I % TILE) return exl_set_err(EXL_ERR_ARG, "decode_plan: widths must be multiples of 128 (hidden of 512): hidden %d attn %d inter %d", H, HQ, I);
    const int gs = q0->groupsize;
    int gs32 = gs / 32, sh = 0;
    if (q0->groups > 1) {
        if (gs % 32 || (gs32 & (gs32 - 1))) return exl_set_err(EXL_ERR_ARG, "decode_plan: groupsize %d must be 32 * 2^n", gs);
        while ((1 << sh) < gs32) sh++;
    } else sh = 30;
    std::vector<LayerDesc> L((size_t)d->n_layers);
    bool any_act = false;
    const int expectK[7] = {H, H, H, HQ, H, H, I}, expectN[7] = {HQ, HQ, HQ, H, I, I, H};
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
    a.n_layers = d->n_layers; a.H = H; a.HQ = HQ; a.I = I; a.heads = d->num_heads; a.max_seq = d->max_seq_len; a.gshift = sh;
    a.eps = d->rms_eps; a.sin = (const half*)d->sin; a.cos = (const half*)d->cos;
    a.final_norm = (const half*)d->final_norm; a.lm_head = (const half*)d->lm_head; a.vocab = d->lm_head ? d->vocab : 0;
    if (d->lm_head && (!d->final_norm || d->vocab % 4)) return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan: lm_head needs final_norm and vocab %% 4 == 0"));
    a.spt_max = spt_max_for(H, HQ, I);
    a.act = any_act ? 1 : 0;
    if (any_act && d->tp_world > 1)
        return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan: act-order matrices under tensor parallelism are not supported by the fused step (o_proj needs the all-gathered attention output): use the per-op path"));
    int dev_smem = 0;
    cudaDeviceGetAttribute(&dev_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, p->device);
    const size_t fixed = smem_fixed_bytes(H, HQ, I, any_act);
    int depth = ring_depth_for((size_t)dev_smem, fixed);
    if (const char* e = getenv("EXL_DS_DEPTH")) { int v = atoi(e); if (v >= 1 && v < depth) depth = v; }
    if (depth < 2) return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan: model too wide for the shared-memory plan (%d ring stages per pipeline)", depth));
    if (d->num_heads > ds->num_sms || d->num_heads > DS_MAX_HEADS) return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan: more heads (%d) than SMs (or than %d)", d->num_heads, DS_MAX_HEADS));
    a.depth = depth;
    p->smem = smem_dynamic_bytes(fixed, depth);
    if ((size_t)H * 2 > (size_t)a.spt_max * 256) return plan_fail(p, exl_set_err(EXL_ERR_ARG, "decode_plan: internal: head staging does not fit"));
    const void* kfn = step_kernel_for(any_act, d->tp_world > 1);
    cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem);
    if (e != cudaSuccess) return plan_fail(p, exl_set_err(EXL_ERR_CUDA, "decode_plan: smem attribute (%zu B): %s", p->smem, cudaGetErrorString(e)));
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kfn, DS_THREADS, p->smem);
    if (e != cudaSuccess || per_sm < 1) return plan_fail(p, exl_set_err(EXL_ERR_CUDA, "decode_plan: kernel does not fit an SM (smem %zu)", p->smem));
    p->grid = ds->num_sms;
    if (const char* eg = getenv("EXL_DS_GRID")) { int v = atoi(eg); if (v >= 1 && v <= ds->num_sms) p->grid = v; }
    a.att_slots = att_slots_for(p->grid, d->num_heads);
    // scratch: accumulators | attention partials | barrier
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
    const size_t o_qkv = take((size_t)3 * HQ * 4), o_o = take((size_t)H * 4), o_gu = take((size_t)2 * I * 4), o_d = take((size_t)H * 4);
    const size_t o_att = take((size_t)d->num_heads * a.att_slots * PART_LD * 4), o_bar = take(256), o_av = take((size_t)HQ * 2);
    const bool want_trace = getenv("EXL_DS_TRACE") != nullptr;
    const size_t o_trace = want_trace ? take((size_t)p->grid * TRACE_LAYERS * 24 * 8) : 0;
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
    if (barriers_per_step) *barriers_per_step = 1 + (5 + (p->args.act ? 1 : 0) + (p->args.tp_world > 1 ? (p->args.tp_reduce ? 4 : 2) : 0)) * (int64_t)p->args.n_layers;
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

extern "C" int exl_decode_step(exl_decode_plan* p, const void* x_in, int past_len, void* x_out, void* logits, void* stream_)
{
    if (!p) return exl_set_err(EXL_ERR_STATE, "decode_step: NULL plan");
    if (!x_in) return exl_set_err(EXL_ERR_ARG, "decode_step: x_in is NULL");
    if (past_len < 0 || past_len >= p->args.max_seq) return exl_set_err(EXL_ERR_ARG, "decode_step: past_len %d outside the cache (max_seq %d)", past_len, p->args.max_seq);
    if (p->args.lm_head && !logits) return exl_set_err(EXL_ERR_ARG, "decode_step: the plan has an lm_head, logits must be given");
    if (!p->peers_ready) return exl_set_err(EXL_ERR_STATE, "decode_step: tensor-parallel plan: call exl_decode_plan_ipc_import first");
    DeviceGuard guard(p->device);
    StepArgs a = p->args;
    a.x_in = (const half*)x_in; a.x_out = (half*)x_out; a.logits = (float*)logits; a.past_len = past_len;
    if (att_needs_reset(a.heads, past_len, p->grid)) {
        // short context: some CTAs inside a head's CTA range own no attention unit in this launch (stateless test, so a captured
        // CUDA graph -- past_len is baked into it -- replays the same decision)
        const int n = a.heads * a.att_slots * PART_LD;
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
    cudaError_t e = cudaLaunchKernelExC(&cfg, step_kernel_for(a.act != 0, a.tp_world > 1), kargs);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    if (e != cudaSuccess) return exl_set_err(EXL_ERR_CUDA, "launch of decode_step_kernel failed: %s (grid %d, smem %zu)", cudaGetErrorString(e), p->grid, p->smem);
    return EXL_OK;
}
