// decode_step_sched.h -- the static work schedule of decode_step_kernel (decode_step.cu): which units of a phase a CTA owns,
// which CTA owns a unit, how many CTAs take part, and the host-side sizing that depends on it.
//
// Plain C++ with no CUDA types: the kernel includes it as device code, and tests/test_decode_schedule.py compiles the same
// header with g++ (tests/decode_sched_check.cpp) to check the partition invariants for every BASELINE shape, tensor-parallel
// shard and context length on the CPU -- a schedule mistake on the GPU is a trapped launch, so it is worth proving first.
#pragma once
#include <cstddef>
#include <type_traits>
#include <utility>

#if defined(__CUDACC__)
#define DS_HD __host__ __device__ __forceinline__
#else
#define DS_HD static inline
#endif

namespace ds_sched {

constexpr int TILE = 128;                        // columns per tile == K rows per stage
constexpr int W_BYTES = 8192;                    // packed weights of one unit: 16 k8-rows x 128 columns x 4 B
constexpr int STAGE_STRIDE = W_BYTES + 2048;     // ring stage: weights + scale rows + zero rows, 1 KB aligned (swizzle atom)
constexpr int PART_LD = 132;                     // attention partial: o[128], m, l, pad
constexpr int MAX_DEPTH = 6;                     // ring stages per pipeline
constexpr int ATT_CTAS_PER_HEAD = 7;             // at most this many CTAs share one head in the attention phase (when heads are few)
constexpr int ATT_CTAS_PER_KV_HEAD = 16;         // the same cap under grouped-query attention, per KV head (a unit does n_rep heads' math)
constexpr int MAX_BATCH = 4;                     // sequences per launch: 8 B columns of the GEMV MMA = 4 sequences x 2 x planes
constexpr int DS_MAX_HEADS = 256;                // (virtual) heads a plan may have: size of the per-head CTA-range table

enum { PH_QKV = 0, PH_ATT = 1, PH_O = 2, PH_GU = 3, PH_DOWN = 4, PH_HEAD = 5 };

// contiguous share of n items for CTA c of G
DS_HD int share_lo(long long n, int c, int G) { return (int)(n * c / G); }
// share of CTA c in a phase that p_G <= G CTAs take part in: [lo, hi), empty for c >= p_G
DS_HD int range_lo(long long n, int c, int pG) { return c >= pG ? (int)n : (int)(n * c / pG); }
// the CTA whose share contains item u (inverse of share_lo)
DS_HD int cta_of(long long u, long long U, int G) { return (int)(((u + 1) * G - 1) / U); }

// U: units; spt: K stages per tile; tpm: tiles per matrix (ATT: units per KV head); tq: tiles of the first matrix (QKV: q is wider than
// k and v under grouped-query attention; every other phase: tpm); G: CTAs that take part in the phase.  Tiles are numbered matrix by
// matrix, so the phase accumulator of tile t starts at column t * TILE ([HQ | HKV | HKV] for QKV, [I | I] for GU).
struct Phase { int kind, U, spt, tpm, tq, nmat, mat0, N, G; float* acc; };

// CTAs that may share one KV head's attention units
DS_HD int att_cap(int heads, int kv_heads) { return kv_heads < heads ? ATT_CTAS_PER_KV_HEAD : ATT_CTAS_PER_HEAD; }

// KV heads and k / v width of a shape: its kv_heads / HKV fields, or heads / HQ (multi-head attention) for a shape type that has none
template <class A, class = void> struct has_kv_heads : std::false_type {};
template <class A> struct has_kv_heads<A, std::void_t<decltype(std::declval<const A&>().kv_heads)>> : std::true_type {};
template <class A> DS_HD int kv_heads_of(const A& a) { if constexpr (has_kv_heads<A>::value) return a.kv_heads; else return a.heads; }
template <class A> DS_HD int hkv_of(const A& a) { if constexpr (has_kv_heads<A>::value) return a.HKV; else return a.HQ; }

// A: anything with the fields H, HQ, I, heads, past_len, vocab, lm_head, acc_qkv, acc_o, acc_gu, acc_d, and for grouped-query
// attention kv_heads and HKV (the kernel's StepArgs).
// nb: sequences in the launch.  The GEMV phases do not depend on it (every sequence rides in the same MMAs).  ATT runs over virtual
// heads: a virtual KV head is (sequence b, KV head kvh) = b * kv_heads + kvh, and past_len is the LONGEST context of the batch (a
// chunk past a shorter sequence's end is an empty unit).
template <class A>
DS_HD Phase phase_of(const A& a, int kind, int grid, int nb = 1)
{
    Phase p; p.kind = kind; p.acc = nullptr; p.G = grid; p.spt = 0; p.tpm = 0; p.tq = 0; p.nmat = 0; p.mat0 = 0; p.N = 0; p.U = 0;
    if (kind == PH_QKV)       { p.spt = a.H / TILE;  p.N = a.HQ; p.nmat = 3; p.mat0 = 0; p.acc = a.acc_qkv; }
    else if (kind == PH_O)    { p.spt = a.HQ / TILE; p.N = a.H;  p.nmat = 1; p.mat0 = 3; p.acc = a.acc_o; }
    else if (kind == PH_GU)   { p.spt = a.H / TILE;  p.N = a.I;  p.nmat = 2; p.mat0 = 4; p.acc = a.acc_gu; }
    else if (kind == PH_DOWN) { p.spt = a.I / TILE;  p.N = a.H;  p.nmat = 1; p.mat0 = 6; p.acc = a.acc_d; }
    if (kind == PH_ATT) {
        const int nch = (a.past_len + 15) >> 4;
        p.tpm = nch > 0 ? nch : 1;                          // units per KV head (one empty unit when there is no history)
        p.tq = p.tpm;
        const int kvh = nb * kv_heads_of(a);
        p.U = kvh * p.tpm;
        // at most ~7 CTAs per head: the O prologue combines one partial per CTA and head (two rounds of 4 loads); with few heads
        // per GPU (tensor parallel) the rest of the grid sits this phase out -- its bytes are small then.  Grouped-query attention:
        // one unit carries the math of n_rep query heads, so up to 16 CTAs share a KV head (70B: 128 of 132 CTAs instead of 56)
        const int cap = att_cap(nb * a.heads, kvh);
        if (kvh * cap < grid) p.G = kvh * cap;
    } else if (kind == PH_HEAD) {
        p.U = a.lm_head ? (int)(((long long)a.vocab * a.H * 2 + W_BYTES - 1) / W_BYTES) : 0;
    } else {
        p.tpm = p.N / TILE;
        p.tq = p.tpm;
        if (kind == PH_QKV) { p.tq = a.HQ / TILE; p.tpm = hkv_of(a) / TILE; }          // q, then k and v (as wide as q unless GQA)
        p.U = (p.tq + (p.nmat - 1) * p.tpm) * p.spt;
    }
    return p;
}
// matrix (0 .. nmat - 1) of tile t of a GEMV phase, its first tile, and its tile count
DS_HD int mat_of_tile(const Phase& p, int t) { return t < p.tq ? 0 : 1 + (t - p.tq) / p.tpm; }
DS_HD int mat_tile0(const Phase& p, int mi) { return mi == 0 ? 0 : p.tq + (mi - 1) * p.tpm; }
DS_HD int mat_tiles(const Phase& p, int mi) { return mi == 0 ? p.tq : p.tpm; }

// Grouped-query attention scratch (decode_step.cu), aliased onto the x staging area, which is dead between the end of the QKV GEMV
// and the O prologue: per (KV-head segment, query head of the group) 4 pipeline partials + the new token's partial and q in fp16;
// per segment the new k and v rows in fp32.  Partials start at offset 0.
DS_HD int gqa_qh_off(int n_rep) { return 2 * n_rep * 5 * PART_LD * 4; }
DS_HD int gqa_kn_off(int n_rep) { return gqa_qh_off(n_rep) + 2 * n_rep * TILE * 2; }
DS_HD int gqa_scratch_bytes(int n_rep) { return n_rep > 1 ? gqa_kn_off(n_rep) + 2 * 2 * TILE * 4 : 0; }
// bytes of the x staging area (quantised x planes + segment table), at least the grouped-query attention scratch
DS_HD int stage_area_bytes(int xstages, int n_rep)
{
    const int b = xstages * (256 + 32), g = gqa_scratch_bytes(n_rep);
    return b > g ? b : ((g + 31) & ~31);
}
// Multi-token plans (ntok consecutive tokens of one sequence) run the grouped-query attention path for any n_rep: a KV head's stage
// serves its n_rep * ntok query vectors (token t, query head r of the group at t * n_rep + r), and the segment keeps the ntok new k
// and v rows in fp32 ([2][ntok][128] each) -- the launch's own tokens are the causal tail of every query vector.
DS_HD int gqa_scratch_bytes_multi(int n_rep, int ntok) { return gqa_kn_off(n_rep * ntok) + 2 * 2 * ntok * TILE * 4; }
DS_HD int stage_area_bytes_multi(int xstages, int n_rep, int ntok)
{
    const int b = xstages * (256 + 32), g = gqa_scratch_bytes_multi(n_rep, ntok);
    return b > g ? b : ((g + 31) & ~31);
}
// The multi-token ATT phase: (KV head, 16-position chunk) units over the kv_heads real KV heads at the shared context past_len (the
// history every token of the launch attends), and the grouped-query cap on CTAs per KV head -- a unit does the math of n_rep * ntok
// query vectors.  Every other phase is phase_of's (the GEMV phases do not depend on the token count; HEAD neither).
template <class A>
DS_HD Phase phase_of_multi(const A& a, int kind, int grid)
{
    Phase p = phase_of(a, kind, grid);
    if (kind == PH_ATT) {
        p.G = grid;
        const int kvh = kv_heads_of(a);
        if (kvh * ATT_CTAS_PER_KV_HEAD < grid) p.G = kvh * ATT_CTAS_PER_KV_HEAD;
    }
    return p;
}

// ---- host side (exl_decode_plan_create / exl_decode_step) ----
// Short contexts: with fewer attention units than participating CTAs (U < G) some CTAs between the first and the last CTA of a
// head own nothing, so the slot they would have written keeps whatever an EARLIER launch left there (a longer context fills
// every slot) -- and the O prologue combines slots [0, c_hi - c_lo] of the head.  exl_decode_step resets the table to the
// neutral partial (m = -inf, l = 0, o = 0) before such a launch.  With one unit per head (tpm == 1) a head has one slot: no gap.
// tests/decode_sched_check.cpp (tests/decode_sched_check_gqa.cpp for GQA) proves: a gap exists only where this predicate holds.
// Grouped-query attention: the same holds per KV head (every query head of the group has the CTA range of its KV head).
// Batched decode: the same over virtual heads, with past_len the longest context of the batch.
struct AttDims { int H, HQ, HKV, I, heads, kv_heads, past_len, vocab; const void* lm_head; float *acc_qkv, *acc_o, *acc_gu, *acc_d; };
static inline bool att_needs_reset(int heads, int kv_heads, int past_len, int grid, int bsz = 1)
{
    AttDims a = {};
    a.heads = heads; a.kv_heads = kv_heads; a.past_len = past_len;
    const Phase p = phase_of(a, PH_ATT, grid, bsz);
    return p.U < p.G && p.tpm >= 2;
}
static inline bool att_needs_reset(int heads, int past_len, int grid) { return att_needs_reset(heads, heads, past_len, grid); }

// slots of att_part per query head: one per CTA that can hold a piece of its KV head (+ 2: a range may start and end inside the head).
// A batch has more virtual heads, so never more CTAs per head: the single-sequence count serves every batch size.
static inline int att_slots_for(int grid, int heads, int kv_heads)
{
    const int cap = att_cap(heads, kv_heads);
    return (grid < cap * kv_heads ? grid / kv_heads : cap) + 2;
}
static inline int att_slots_for(int grid, int heads) { return att_slots_for(grid, heads, heads); }
static inline int spt_max_for(int H, int HQ, int I)
{
    int m = (H > I ? H : I) / TILE;
    return HQ / TILE > m ? HQ / TILE : m;
}
constexpr size_t SMEM_STATIC_ALLOWANCE = 2048;   // static __shared__ of the kernel (mbarriers, schedule tables): ptxas reports 1664 B (1920 B for the batched kernels)
// Batched plans stage x compacted: a CTA keeps only the K stages it quantises (s_rng[.][3] = min(share, spt)) per sequence, not
// spt_max of them.  The area per sequence also holds the head's normalised x (H fp16 = H / 128 stages' bytes).
static inline int batch_xstages(int H, int HQ, int HKV, int I, int grid)
{
    AttDims a = {};
    a.H = H; a.HQ = HQ; a.HKV = HKV; a.I = I; a.heads = HQ / TILE; a.kv_heads = HKV / TILE;
    int m = H / TILE;
    const int kinds[4] = {PH_QKV, PH_O, PH_GU, PH_DOWN};
    for (int k = 0; k < 4; k++) {
        const Phase p = phase_of(a, kinds[k], grid);
        const int share = (p.U + p.G - 1) / p.G;             // the largest share of a CTA
        const int n = share < p.spt ? share : p.spt;
        if (n > m) m = n;
    }
    return m;
}
// shared memory apart from the ring: alignment slack, x staging (+ a second slot of H / 128 stages with act-order; grouped-query
// attention scratch shares it), residual stream, attention scratch (partials, q / new k / new v in fp32, q in fp16), norm weights,
// static variables.  max_batch > 1 (no act-order): max_batch x xstages compacted stages (batch_xstages) and max_batch residual
// streams; the attention scratch is per head segment and does not grow.  max_batch == 1 is the single-sequence plan.
static inline size_t smem_fixed_bytes(int H, int HQ, int I, bool act, int n_rep = 1, int max_batch = 1, int xstages = 0)
{
    const size_t tail = (size_t)(2 * 17 * PART_LD + 6 * TILE) * 4 + (size_t)2 * TILE * 2 /* fp16 q */ + (size_t)H * 2 /* wnorm */ + SMEM_STATIC_ALLOWANCE;
    if (max_batch > 1) return 1024 + (size_t)stage_area_bytes(max_batch * xstages, n_rep) + (size_t)max_batch * H * 2 + tail;
    return 1024 + (size_t)stage_area_bytes(spt_max_for(H, HQ, I) + (act ? H / TILE : 0), n_rep) + (size_t)H * 2 + tail;
}
// dynamic shared memory to request for `depth` ring stages per pipeline
static inline size_t smem_dynamic_bytes(size_t fixed, int depth) { return fixed - SMEM_STATIC_ALLOWANCE + (size_t)4 * depth * STAGE_STRIDE; }
// ring stages per pipeline that fit (0: the model is too wide)
static inline int ring_depth_for(size_t dev_smem, size_t fixed)
{
    if (dev_smem <= fixed) return 0;
    int depth = (int)((dev_smem - fixed) / STAGE_STRIDE) / 4;
    return depth > MAX_DEPTH ? MAX_DEPTH : depth;
}
// The largest batch (<= MAX_BATCH) a plan can take: >= 2 ring stages per pipeline, at most 2 head segments per CTA in ATT (every
// virtual head -- virtual KV head under grouped-query attention -- needs a CTA of its own: max_batch * heads <= grid), and the
// per-head CTA-range table.  Act-order plans take one sequence.  0: not even one fits.
static inline int max_batch_for(int H, int HQ, int I, int heads, int kv_heads, bool act, size_t dev_smem, int grid)
{
    const int n_rep = heads / kv_heads;
    const int xst = batch_xstages(H, HQ, kv_heads * TILE, I, grid);
    int best = 0;
    for (int b = 1; b <= (act ? 1 : MAX_BATCH); b++) {
        if (b * (n_rep > 1 ? kv_heads : heads) > grid || b * heads > DS_MAX_HEADS) break;
        if (ring_depth_for(dev_smem, smem_fixed_bytes(H, HQ, I, act, n_rep, b, xst)) < 2) break;
        best = b;
    }
    return best;
}

// ---- multi-token plans (exl_decode_plan_create_multi / exl_decode_step_multi): 1 .. max_tokens consecutive tokens of ONE sequence ----
// The GEMV, norm and head phases are the batch's with nb = n tokens; ATT is phase_of_multi's.  Its slot table, reset predicate and
// shared memory follow.  tests/decode_sched_check_multi.cpp proves them for every token count and context.
// Exact: with fewer units than CTAs every CTA holds at most one unit, so a KV head's range has an idle CTA exactly when it spans more
// CTAs than the head has units (the plain U < G test also fires at contexts where every range happens to be dense).
static inline bool att_needs_reset_multi(int heads, int kv_heads, int past_len, int grid)
{
    AttDims a = {};
    a.heads = heads; a.kv_heads = kv_heads; a.past_len = past_len;
    const Phase p = phase_of_multi(a, PH_ATT, grid);
    if (p.U >= p.G || p.tpm < 2) return false;
    for (int kvh = 0; kvh < kv_heads; kvh++)
        if (cta_of((long long)(kvh + 1) * p.tpm - 1, p.U, p.G) - cta_of((long long)kvh * p.tpm, p.U, p.G) + 1 > p.tpm) return true;
    return false;
}
// slots of att_part per virtual query head (token t, head h): one per CTA that can hold a piece of its KV head, + 2
static inline int att_slots_multi(int grid, int kv_heads)
{
    return (grid < ATT_CTAS_PER_KV_HEAD * kv_heads ? grid / kv_heads : ATT_CTAS_PER_KV_HEAD) + 2;
}
// as smem_fixed_bytes for a batch of max_tokens, with the multi-token attention scratch sharing the staging area
static inline size_t smem_fixed_bytes_multi(int H, int n_rep, int max_tokens, int xstages)
{
    const size_t tail = (size_t)(2 * 17 * PART_LD + 6 * TILE) * 4 + (size_t)2 * TILE * 2 /* fp16 q */ + (size_t)H * 2 /* wnorm */ + SMEM_STATIC_ALLOWANCE;
    return 1024 + (size_t)stage_area_bytes_multi(max_tokens * xstages, n_rep, max_tokens) + (size_t)max_tokens * H * 2 + tail;
}
// The most tokens (<= MAX_BATCH) a multi-token plan can take: >= 2 ring stages per pipeline, every KV head a CTA of its own (at most 2
// head segments per CTA), and max_tokens * heads virtual query heads in the CTA-range table.  0: not even one fits.
static inline int max_tokens_for(int H, int HQ, int I, int heads, int kv_heads, size_t dev_smem, int grid)
{
    const int xst = batch_xstages(H, HQ, kv_heads * TILE, I, grid);
    int best = 0;
    for (int k = 1; k <= MAX_BATCH; k++) {
        if (kv_heads > grid || k * heads > DS_MAX_HEADS) break;
        if (ring_depth_for(dev_smem, smem_fixed_bytes_multi(H, heads / kv_heads, k, xst)) < 2) break;
        best = k;
    }
    return best;
}

// ---- LoRA adapters (exl_decode_plan_create_lora) ----
// An adapted phase (any of its matrices has rank > 0) gets one extra step after its prologue, LA: units (adapted matrix j of the phase,
// 128-row K stage s), numbered j * spt + s and cut into G contiguous shares.  The CTA of a unit dots that K stage of x with the 128 rows
// of A and adds the result into t[b][rank] in L2; one grid barrier then makes t complete.  In the GEMV the B term of a tile of an
// adapted matrix is added by exactly one CTA: the one that owns the tile's K stage 0.  A and B are read from global memory by the
// consumers (no ring stage, no shared memory beyond the attention partial area, which is free outside ATT).
constexpr int LORA_MAX_RANK = 128;
DS_HD bool lora_rank_ok(int r) { return r >= 0 && r <= LORA_MAX_RANK && r % 8 == 0; }
DS_HD int lora_units(int n_adapted, int spt) { return n_adapted * spt; }
// the CTA that adds the B term of tile `tile` of a GEMV phase
DS_HD int lora_b_cta(const Phase& p, int tile) { return cta_of((long long)tile * p.spt, p.U, p.G); }
// first tile whose K stage 0 lies in the unit range [u0, u1) of a CTA (the B-term tiles are [first, last] with last = (u1 - 1) / spt)
DS_HD int lora_b_first(const Phase& p, int u0) { return (u0 + p.spt - 1) / p.spt; }
// fp32 floats of the LA step's shared scratch: x of one K stage and the partial t, per sequence (it lives in the attention partials)
DS_HD int lora_scratch_floats(int max_batch, int max_rank) { return max_batch * (TILE + max_rank); }
constexpr int LORA_SCRATCH_ROOM = 2 * 17 * PART_LD;
// phase of matrix m (q k v o gate up down)
DS_HD int lora_phase_of_mat(int m) { return m < 3 ? PH_QKV : (m == 3 ? PH_O : (m < 6 ? PH_GU : PH_DOWN)); }
// extra grid barriers per step: one per adapted phase of every layer; rank: [n_layers * 7]
static inline long long lora_barriers(const int* rank, int n_layers)
{
    long long n = 0;
    for (int l = 0; l < n_layers; l++) {
        bool ph[6] = {false, false, false, false, false, false};
        for (int m = 0; m < 7; m++) if (rank[l * 7 + m] > 0) ph[lora_phase_of_mat(m)] = true;
        n += (int)ph[PH_QKV] + (int)ph[PH_O] + (int)ph[PH_GU] + (int)ph[PH_DOWN];
    }
    return n;
}

} // namespace ds_sched
