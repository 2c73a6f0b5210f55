// logprob.cu -- exl_token_logprobs: per-token log-probabilities and greedy ids of given targets, lm_head GEMM and log-softmax fused,
// without writing the logits.  The reference computes matmul(hn, lm_head^T).float() over every position and then log_softmax +
// gather in torch (perplexity.py:118-121), materialising [T, vocab] three times.
//
//   logit[t, v]  = sum_k hn[t, k] * lm_head[v, k]     fp32 accumulation of exact fp16 products (the decode step's HEAD convention)
//   logprob[t]   = logit[t, targets[t]] - logsumexp_v logit[t, v]
//   greedy[t]    = argmax_v logit[t, v], ties to the lower id
//
// Launch 1, token_logprob_kernel: one CTA per (row tile, vocab chunk) of logprob_sched.h.
//   warp 8     TMA producer: per 64-wide k-block the 128 x 64 tile of hn and the 256 x 64 tile of lm_head (both K-major, SWIZZLE_128B)
//              into a 4-stage ring, over every vocab tile of the chunk in turn
//   warps 0-7  two warpgroups, rows [64 wg, 64 wg + 64) of the tile: wgmma m64n256k16, fp32 accumulators in registers.  After the
//              last k-block of a vocab tile each thread folds its 2 rows x 64 columns into its running (max, sum of exp, argmax,
//              target logit); ids >= V (the TMA zero fill of the last tile) count as -inf.  At the end of the chunk the four threads
//              of a quad (which hold all columns of their rows) merge, and one writes the row's partial to work[t][chunk].
// Launch 2, logprob_combine_kernel: one thread per row merges the row's partials in chunk order (float64).
// No atomics and no allocation: two calls are bitwise equal, and the call can be captured in a CUDA graph.
#include "exl_common.cuh"
#include "logprob_sched.h"
#include <cmath>

namespace {

using lp_sched::BM;
using lp_sched::BN;
using lp_sched::BK;

constexpr int A_BYTES = BM * BK * 2;          // 16 KB: hn tile, K-major SW128
constexpr int B_BYTES = BN * BK * 2;          // 32 KB: lm_head tile, K-major SW128
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int NSTAGE = 4;
constexpr int CONSUMERS = 256;
constexpr int LP_THREADS = CONSUMERS + 32;
constexpr size_t LP_SMEM = 1024 + (size_t)NSTAGE * STAGE_BYTES;
static_assert(sizeof(float4) == lp_sched::PART_BYTES, "a partial is one float4");

struct alignas(64) LpArgs
{
    CUtensorMap tmap_a;      // hn      [T, H] fp16, box 64 (k) x 128 (rows)
    CUtensorMap tmap_b;      // lm_head [V, H] fp16, box 64 (k) x 256 (ids)
    const int64_t* targets;
    float4* part;            // [T][chunks] {max, sum exp(logit - max), argmax (int bits), target logit or -inf}
    lp_sched::Plan plan;
    int H;
};

__device__ __forceinline__ uint32_t s_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_init(void* b, int c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(s_u32(b)), "r"(c)); }
__device__ __forceinline__ void bar_expect_tx(void* b, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(s_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bar_arrive(void* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(s_u32(b)) : "memory"); }
__device__ __forceinline__ void bar_wait(void* b, uint32_t parity)
{
    asm volatile("{\n\t.reg .pred p;\n\tLP_WAIT:\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                 "@p bra LP_DONE;\n\tbra LP_WAIT;\n\tLP_DONE:\n\t}" :: "r"(s_u32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_2d(void* dst, const CUtensorMap* tm, int c0, int c1, void* bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 :: "r"(s_u32(dst)), "l"(tm), "r"(c0), "r"(c1), "r"(s_u32(bar)) : "memory");
}
// wgmma shared-memory descriptor, K-major, SWIZZLE_128B: start >> 4 | LBO (unused) | SBO = 1024 B (8 rows x 128 B) | 128B swizzle
__device__ __forceinline__ uint64_t desc_sw128(uint32_t smem_addr)
{
    return (uint64_t)((smem_addr & 0x3ffffu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// D[64 x 256] (+)= A[64 x 16] . B[256 x 16]^T, both K-major in shared memory; scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t scale_d)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, "
                 "%128, %129, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
                 : "l"(adesc), "l"(bdesc), "r"(scale_d) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N_> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N_) : "memory"); }

// one row's running state over the vocab tiles a thread has seen
struct RowState { float m; double s; int arg; float tgt; int bad; };

__device__ __forceinline__ void row_init(RowState& r) { r.m = -INFINITY; r.s = 0.0; r.arg = 0x7fffffff; r.tgt = -INFINITY; r.bad = 0; }

// fold the 64 logits a thread holds of one row of the tile (columns cb + 8 j + e, j < 32, e < 2; registers 4 j + off + e) into r.
// lim: columns at or past it are ids >= V.  tc: the target's column relative to cb (any value if the target is elsewhere).
template <int OFF>
__device__ __forceinline__ void row_fold(RowState& r, const float (&acc)[128], int cb, int lim, int tc)
{
    float tm = -INFINITY; int ta = 0x7fffffff; int bad = 0; float tg = -INFINITY;
    #pragma unroll
    for (int j = 0; j < 32; j++) {
        #pragma unroll
        for (int e = 0; e < 2; e++) {
            const int c = 8 * j + e;
            const float x = acc[4 * j + OFF + e];
            if (c < lim) {
                bad |= !(fabsf(x) <= 3.402823466e38f);
                if (x > tm) { tm = x; ta = cb + c; }          // columns ascend: strict > keeps the lower id on a tie
                if (c == tc) tg = x;
            }
        }
    }
    const float m = fmaxf(r.m, tm);
    float ts = 0.f;
    #pragma unroll
    for (int j = 0; j < 32; j++) {
        #pragma unroll
        for (int e = 0; e < 2; e++) {
            const int c = 8 * j + e;
            if (c < lim) ts += expf(acc[4 * j + OFF + e] - m);
        }
    }
    if (tm > r.m) r.arg = ta;                                   // earlier tiles hold lower ids: a tie keeps r.arg
    r.s = (r.m == m ? r.s : r.s * (double)expf(r.m - m)) + (double)ts;
    r.m = m;
    r.tgt = fmaxf(r.tgt, tg);
    r.bad |= bad;
}

// merge the states of the four threads of a quad (xor butterfly: every lane ends with the same state)
__device__ __forceinline__ void row_quad_merge(RowState& r)
{
    #pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, r.m, o);
        const double os = __shfl_xor_sync(0xffffffffu, r.s, o);
        const int oa = __shfl_xor_sync(0xffffffffu, r.arg, o);
        const float ot = __shfl_xor_sync(0xffffffffu, r.tgt, o);
        const int ob = __shfl_xor_sync(0xffffffffu, r.bad, o);
        const float m = fmaxf(r.m, om);
        const double a = r.m == m ? r.s : r.s * (double)expf(r.m - m);
        const double b = om == m ? os : os * (double)expf(om - m);
        r.s = r.m < om ? b + a : a + b;                         // the same operand order on both lanes of a pair
        if (om > r.m || (om == r.m && oa < r.arg)) r.arg = oa;
        r.m = m;
        r.tgt = fmaxf(r.tgt, ot);
        r.bad |= ob;
    }
}

__global__ void __launch_bounds__(LP_THREADS, 1) token_logprob_kernel(const __grid_constant__ LpArgs a)
{
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = smem_raw + ((1024u - (s_u32(smem_raw) & 1023u)) & 1023u);
    __shared__ __align__(8) unsigned long long full[NSTAGE], empty[NSTAGE];

    const lp_sched::Plan& p = a.plan;
    const int tid = threadIdx.x, warp = tid >> 5;
    const int rt = lp_sched::row_tile_of(p, blockIdx.x), ch = lp_sched::chunk_of(p, blockIdx.x);
    const int vt0 = lp_sched::chunk_begin(p, ch), vt1 = lp_sched::chunk_begin(p, ch + 1);
    const int r0 = rt * BM;
    const int nkb = a.H / BK;
    const int total = (vt1 - vt0) * nkb;

    if (tid == 0) {
        for (int i = 0; i < NSTAGE; i++) { bar_init(&full[i], 1); bar_init(&empty[i], CONSUMERS / 128); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == CONSUMERS / 32) {
        // ================================ TMA producer ================================
        if ((tid & 31) == 0) {
            for (int it = 0; it < total; it++) {
                const int s = it % NSTAGE, kb = it % nkb, vt = vt0 + it / nkb;
                if (it >= NSTAGE) bar_wait(&empty[s], (uint32_t)((it / NSTAGE) - 1) & 1u);
                unsigned char* st = smem + (size_t)s * STAGE_BYTES;
                bar_expect_tx(&full[s], STAGE_BYTES);
                tma_2d(st, &a.tmap_a, kb * BK, r0, &full[s]);
                tma_2d(st + A_BYTES, &a.tmap_b, kb * BK, vt * BN, &full[s]);
            }
        }
        return;
    }

    // ================================ consumers ================================
    const int wg = tid >> 7, lane = tid & 31, wi = warp & 3;
    const int ra = r0 + wg * 64 + wi * 16 + (lane >> 2), rb = ra + 8;     // this thread's two rows (m64n256 fragment)
    const long long ta = ra < p.T ? (long long)a.targets[ra] : -1, tb = rb < p.T ? (long long)a.targets[rb] : -1;
    RowState sa, sb;
    row_init(sa); row_init(sb);
    const bool leader = (tid & 127) == 0;
    float acc[128];
    int it = 0;                                                // k-blocks consumed so far: ring stage it % NSTAGE
    for (int vt = vt0; vt < vt1; vt++) {
        #pragma unroll
        for (int i = 0; i < 128; i++) acc[i] = 0.f;
        for (int kb = 0; kb < nkb; kb++, it++) {
            const int s = it % NSTAGE;
            unsigned char* st = smem + (size_t)s * STAGE_BYTES;
            bar_wait(&full[s], (uint32_t)(it / NSTAGE) & 1u);
            wgmma_fence();
            const uint32_t a_addr = s_u32(st) + (uint32_t)(wg * 64) * 128u;
            const uint32_t b_addr = s_u32(st + A_BYTES);
            #pragma unroll
            for (int k = 0; k < BK / 16; k++)
                wgmma_m64n256k16(acc, desc_sw128(a_addr + k * 32), desc_sw128(b_addr + k * 32), 1u);
            wgmma_commit();
            wgmma_wait<1>();                                   // the wgmmas of k-block it - 1 are done: release their stage
            if (kb > 0 && leader) bar_arrive(&empty[(it - 1) % NSTAGE]);
        }
        wgmma_wait<0>();
        if (leader) bar_arrive(&empty[(it - 1) % NSTAGE]);
        // fragment: register 4 j + e is row ra, 4 j + 2 + e row rb, both at column v0 + 8 j + 2 (lane % 4) + e
        const int cb = vt * BN + 2 * (lane & 3);
        const int lim = p.V - cb;
        const long long da = ta - cb, db = tb - cb;
        row_fold<0>(sa, acc, cb, lim, (da >= 0 && da < BN) ? (int)da : -1);
        row_fold<2>(sb, acc, cb, lim, (db >= 0 && db < BN) ? (int)db : -1);
    }
    row_quad_merge(sa);
    row_quad_merge(sb);
    if ((lane & 3) == 0) {
        #pragma unroll
        for (int h = 0; h < 2; h++) {
            const RowState& r = h ? sb : sa;
            const int row = h ? rb : ra;
            if (row < p.T)
                a.part[lp_sched::slot(p, row, ch)] = make_float4(r.bad ? __int_as_float(0x7fffffff) : r.m, (float)r.s,
                                                                 __int_as_float(r.arg), r.tgt);
        }
    }
}

// one thread per row: the row's partials in chunk order -> logprob, greedy
__global__ void __launch_bounds__(128) logprob_combine_kernel(const float4* __restrict__ part, const int64_t* __restrict__ targets,
                                                              lp_sched::Plan p, float* __restrict__ logprob, int64_t* __restrict__ greedy)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= p.T) return;
    float m = -INFINITY, tgt = -INFINITY;
    int arg = -1;
    bool bad = false;
    for (int c = 0; c < p.chunks; c++) {
        const float4 q = part[lp_sched::slot(p, t, c)];
        bad |= q.x != q.x;
        if (q.x > m) { m = q.x; arg = __float_as_int(q.z); }    // chunks ascend: the first chunk holding the maximum wins a tie
        tgt = fmaxf(tgt, q.w);
    }
    double s = 0.0;
    for (int c = 0; c < p.chunks; c++) {
        const float4 q = part[lp_sched::slot(p, t, c)];
        s += (double)q.y * exp((double)q.x - (double)m);
    }
    const int64_t y = targets[t];
    const bool in = y >= 0 && y < p.V;
    logprob[t] = (bad || !in) ? __int_as_float(0x7fffffff) : (float)((double)tgt - (double)m - log(s));
    greedy[t] = bad ? -1 : (int64_t)arg;
}

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeFn get_encode()
{
    static EncodeFn encode = nullptr;
    if (!encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            encode = (EncodeFn)fn;
    }
    return encode;
}

int encode_rows(EncodeFn encode, CUtensorMap* tm, const void* base, int rows, int H, int box_rows, const char* what)
{
    const cuuint64_t dims[2] = {(cuuint64_t)H, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)H * 2};
    const cuuint32_t box[2] = {BK, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = encode(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return exl_set_err(EXL_ERR_CUDA, "token_logprobs: tensor map for %s failed (%d)", what, (int)r);
    return EXL_OK;
}

// device of a device pointer, or -1 (host memory, unknown pointer, no GPU)
int device_of(const void* ptr)
{
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, ptr) != cudaSuccess) { cudaGetLastError(); return -1; }
    return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged ? at.device : -1;
}

bool g_lp_attr[EXL_MAX_DEVICES];

} // namespace

extern "C" {

int exl_token_logprobs_work_size(int T, int V, int device, int64_t* bytes)
{
    if (!bytes) return exl_set_err(EXL_ERR_ARG, "token_logprobs_work_size: bytes is NULL");
    if (T < 1 || V < 1) return exl_set_err(EXL_ERR_ARG, "token_logprobs_work_size: T %d and V %d must be at least 1", T, V);
    ExlDevice* ds = exl_device_state(device);
    if (!ds) return EXL_ERR_CUDA;
    *bytes = lp_sched::work_bytes(lp_sched::make_plan(T, V, ds->num_sms));
    return EXL_OK;
}

int exl_token_logprobs(const void* hn, int T, int H, const void* lm_head, int V, const int64_t* targets, float* logprob,
                       int64_t* greedy, void* work, int64_t work_bytes, void* stream_)
{
    if (T < 1 || V < 1) return exl_set_err(EXL_ERR_ARG, "token_logprobs: T %d and V %d must be at least 1", T, V);
    if (H < BK || H % BK != 0) return exl_set_err(EXL_ERR_ARG, "token_logprobs: H %d is not a positive multiple of %d", H, BK);
    const void* ptrs[6] = {hn, lm_head, targets, logprob, greedy, work};
    const char* names[6] = {"hn", "lm_head", "targets", "logprob", "greedy", "work"};
    for (int i = 0; i < 6; i++)
        if (!ptrs[i] || ((uintptr_t)ptrs[i] & 15u))
            return exl_set_err(EXL_ERR_ARG, "token_logprobs: %s %p is NULL or not 16-byte aligned", names[i], ptrs[i]);
    const int dev = device_of(hn);
    if (dev < 0) {
        int count = 0;
        if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
            cudaGetLastError();
            return exl_set_err(EXL_ERR_CUDA, "token_logprobs: no CUDA device available; libexl_b200 has no CPU fallback");
        }
        return exl_set_err(EXL_ERR_ARG, "token_logprobs: hn %p is not device memory", hn);
    }
    for (int i = 1; i < 6; i++) {
        const int d = device_of(ptrs[i]);
        if (d != dev) return exl_set_err(EXL_ERR_ARG, "token_logprobs: %s is on device %d, hn on device %d", names[i], d, dev);
    }
    ExlDevice* ds = exl_device_state(dev);
    if (!ds) return EXL_ERR_CUDA;
    const lp_sched::Plan plan = lp_sched::make_plan(T, V, ds->num_sms);
    const long long need = lp_sched::work_bytes(plan);
    if (work_bytes < need)
        return exl_set_err(EXL_ERR_ARG, "token_logprobs: work_bytes %lld < %lld (exl_token_logprobs_work_size)", (long long)work_bytes, need);
    EncodeFn encode = get_encode();
    if (!encode) return exl_set_err(EXL_ERR_CUDA, "token_logprobs: cuTensorMapEncodeTiled unavailable");

    DeviceGuard guard(dev);
    cudaStream_t stream = (cudaStream_t)stream_;
    LpArgs a;
    memset(&a, 0, sizeof(a));
    int rc = encode_rows(encode, &a.tmap_a, hn, T, H, BM, "hn");
    if (rc != EXL_OK) return rc;
    rc = encode_rows(encode, &a.tmap_b, lm_head, V, H, BN, "lm_head");
    if (rc != EXL_OK) return rc;
    a.targets = targets; a.part = (float4*)work; a.plan = plan; a.H = H;
    if (!g_lp_attr[dev]) {
        EXL_CUDA_TRY(cudaFuncSetAttribute(token_logprob_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LP_SMEM));
        g_lp_attr[dev] = true;
    }
    token_logprob_kernel<<<(unsigned)lp_sched::ctas(plan), LP_THREADS, LP_SMEM, stream>>>(a);
    EXL_CHECK_LAUNCH("token_logprob_kernel");
    logprob_combine_kernel<<<(unsigned)((T + 127) / 128), 128, 0, stream>>>((const float4*)work, targets, plan, logprob, greedy);
    EXL_CHECK_LAUNCH("logprob_combine_kernel");
    return EXL_OK;
}

} // extern "C"
