// q4_gemm_tc.cu -- prefill hot path: GPTQ 4-bit fused-dequant GEMM on the Hopper tensor cores (wgmma).
//
//   out[M, N] (=|+=) x[M, K] . W[K, N],   W[k, n] = scales[g(k), n] * (q[k, n] - (zeros[g(k), n] + 1))
//
// Replaces the reference's prefill path -- column_remap + Q4Matrix::reconstruct (a full fp16 copy of W written to and
// re-read from HBM) + cublasHgemm (exllama_ext/cuda_func/q4_matmul.cu:301-344, q4_matrix.cu:170-223) -- with one
// kernel that never materialises W:
//
//   warp 8     TMA producer: per 64-wide k-block MT 128 x 64 fp16 tiles of x (SWIZZLE_128B, K-major as wgmma reads it) and
//              the matching 8 x 128 tile of packed qweight words into a 4-stage smem ring
//   warps 0-7  two warpgroups: dequantise the packed tile into the B operand (thread = (column n, half of the k-block); value =
//              hmul(half(q - zp), scale), bit-identical to reconstruct_kernel, q4_matrix.cu:196-208), then wgmma.mma_async
//              m64n128k16 on their own rows, fp32 accumulators in registers, epilogue from registers.  B has three buffers: the
//              dequant of k-block kb + 1 overlaps the wgmmas of kb (wgmma.wait_group 1 before the next barrier).
//   With MT = 2 a CTA computes a 256 x 128 tile from ONE dequantised B tile, halving the unpack work per MMA.
//
// Act-order matrices gather the columns of x once per call into the library scratch (exl_column_remap) so the TMA
// tile of x is dense; the gather is 2*M*K bytes against 2*M*K*N flops of GEMM.
// fp32 accumulation of exact fp16 products: at least as accurate as the reference's cublasHgemm.
#include "exl_common.cuh"
#include <cstring>

namespace {

constexpr int BM = 128, BN = 128, BK = 64;    // x sub-tile (rows) x columns x k-block; a CTA owns MT (1 or 2) x sub-tiles
constexpr int A_BYTES = BM * BK * 2;          // 16 KB per x sub-tile, K-major SW128
constexpr int WQ_BYTES = (BK / 8) * BN * 4;   // 4 KB packed words [8][128]
constexpr int B_BYTES = BN * BK * 2;          // 16 KB, K-major SW128
constexpr int NSTAGE = 4;                     // TMA ring: x sub-tiles + packed words
constexpr int NBBUF = 3;                      // dequantised B operand
constexpr int CONSUMERS = 256;                // two warpgroups: dequant + wgmma + epilogue
constexpr int TC_THREADS = CONSUMERS + 32;    // + one TMA producer warp

struct alignas(64) TcArgs
{
    CUtensorMap tmap_x;      // x  [M, K] fp16, box 64 (k) x 128 (m), SWIZZLE_128B
    CUtensorMap tmap_w;      // qw [K/8, N] u32, box 128 (n) x 8 (k8), no swizzle
    const uint32_t* qz; const half* sc; half* out;
    int M, N, K, groups, gs_shift32, no_zero;
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
    asm volatile("{\n\t.reg .pred p;\n\tWAIT_LOOP:\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                 "@p bra DONE;\n\tbra WAIT_LOOP;\n\tDONE:\n\t}" :: "r"(s_u32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_2d(void* dst, const CUtensorMap* tm, int c0, int c1, void* bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 :: "r"(s_u32(dst)), "l"(tm), "r"(c0), "r"(c1), "r"(s_u32(bar)) : "memory");
}
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" :: "n"(CONSUMERS) : "memory"); }
// wgmma shared-memory descriptor, K-major, SWIZZLE_128B: start >> 4 | LBO (unused) | SBO = 1024 B (8 rows x 128 B) | 128B swizzle
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr)
{
    return (uint64_t)((smem_addr & 0x3ffffu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// D[64 x 128] (+)= A[64 x 16] . B[16 x 128]^T: A and B K-major in shared memory, fp32 accumulators in registers (scale_d = 0 overwrites D)
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
                 "%64, %65, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(adesc), "l"(bdesc), "r"(scale_d) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N_> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N_) : "memory"); }

// one packed word -> 8 halves in natural k order, value = hmul(half(q - zp), scale): bit-exact reconstruct_kernel
__device__ __forceinline__ uint4 dequant8(uint32_t w, uint32_t zs, uint32_t zf, uint32_t s2)
{
    const uint32_t MLO = 0x000f000fu, MHI = 0x00f000f0u, EX = 0x64006400u, R16 = 0x2c002c00u;
    uint32_t p04, p15, p26, p37, t;
    const uint32_t w8 = w >> 8;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(t) : "r"(w), "r"(MLO), "r"(EX));  asm("sub.f16x2 %0, %1, %2;" : "=r"(p04) : "r"(t), "r"(zs));
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(t) : "r"(w), "r"(MHI), "r"(EX));  asm("fma.rn.f16x2 %0, %1, %2, %3;" : "=r"(p15) : "r"(t), "r"(R16), "r"(zf));
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(t) : "r"(w8), "r"(MLO), "r"(EX)); asm("sub.f16x2 %0, %1, %2;" : "=r"(p26) : "r"(t), "r"(zs));
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(t) : "r"(w8), "r"(MHI), "r"(EX)); asm("fma.rn.f16x2 %0, %1, %2, %3;" : "=r"(p37) : "r"(t), "r"(R16), "r"(zf));
    uint4 o;
    o.x = __byte_perm(p04, p15, 0x5410);     // {q0, q1}
    o.y = __byte_perm(p26, p37, 0x5410);     // {q2, q3}
    o.z = __byte_perm(p04, p15, 0x7632);     // {q4, q5}
    o.w = __byte_perm(p26, p37, 0x7632);     // {q6, q7}
    asm("mul.f16x2 %0, %1, %2;" : "=r"(o.x) : "r"(o.x), "r"(s2));
    asm("mul.f16x2 %0, %1, %2;" : "=r"(o.y) : "r"(o.y), "r"(s2));
    asm("mul.f16x2 %0, %1, %2;" : "=r"(o.z) : "r"(o.z), "r"(s2));
    asm("mul.f16x2 %0, %1, %2;" : "=r"(o.w) : "r"(o.w), "r"(s2));
    return o;
}

template <int MT>
__global__ void __launch_bounds__(TC_THREADS, 1) q4_gemm_tc_kernel(const __grid_constant__ TcArgs a)
{
    constexpr int STAGE_B = MT * A_BYTES + WQ_BYTES;             // a multiple of 1024: every operand tile stays 1 KB aligned
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = smem_raw + ((1024u - (s_u32(smem_raw) & 1023u)) & 1023u);
    __shared__ __align__(8) unsigned long long full_in[NSTAGE], empty[NSTAGE];
    unsigned char* bbuf = smem + (size_t)NSTAGE * STAGE_B;

    const int tid = threadIdx.x, warp = tid >> 5;
    const int n0 = blockIdx.x * BN, m0 = blockIdx.y * (BM * MT);
    const int nkb = a.K / BK;

    if (tid == 0) {
        for (int i = 0; i < NSTAGE; i++) { bar_init(&full_in[i], 1); bar_init(&empty[i], CONSUMERS / 128); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == CONSUMERS / 32) {
        // ================================ TMA producer ================================
        if ((tid & 31) == 0) {
            for (int kb = 0; kb < nkb; kb++) {
                const int s = kb % NSTAGE;
                if (kb >= NSTAGE) bar_wait(&empty[s], (uint32_t)((kb / NSTAGE) - 1) & 1u);
                unsigned char* st = smem + (size_t)s * STAGE_B;
                bar_expect_tx(&full_in[s], MT * A_BYTES + WQ_BYTES);
                #pragma unroll
                for (int h = 0; h < MT; h++) tma_2d(st + h * A_BYTES, &a.tmap_x, kb * BK, m0 + h * BM, &full_in[s]);   // x tiles: (k, m)
                tma_2d(st + MT * A_BYTES, &a.tmap_w, n0, kb * (BK / 8), &full_in[s]);                                 // packed words: (n, k8)
            }
        }
        return;
    }

    // ================================ consumers ================================
    const int wg = tid >> 7;                       // warpgroup: rows [wg * MT * 64, (wg + 1) * MT * 64) of the CTA tile
    const int cn = tid & (BN - 1);                 // dequant: column inside the tile ...
    const int hh = tid >> 7;                       // ... and half of the k-block (4 words = 32 k)
    const int col = n0 + cn;
    const int colc = col < a.N ? col : (a.N - 1);
    // group parameters are fetched one k-block ahead (raw words in registers) so their L2 latency never sits on the
    // dequant -> MMA critical path
    int cur_grp = -1, nxt_grp = -1;
    uint32_t zs = 0, zf = 0, s2 = 0, nxt_zw = 0; unsigned short nxt_sh = 0;
    const uint32_t b_off = (uint32_t)((cn >> 3) * 1024 + (cn & 7) * 128);
    auto grp_of = [&](int kb) { return a.groups == 1 ? 0 : ((kb * 2 + hh) >> a.gs_shift32); };
    auto fetch = [&](int grp) {
        nxt_zw = __ldg(a.qz + (size_t)grp * (a.N >> 3) + (colc >> 3));
        nxt_sh = __half_as_ushort(__ldg(a.sc + (size_t)grp * a.N + colc));
        nxt_grp = grp;
    };
    fetch(grp_of(0));

    float acc[MT][64];
    #pragma unroll
    for (int h = 0; h < MT; h++) {
        #pragma unroll
        for (int i = 0; i < 64; i++) acc[h][i] = 0.f;
    }

    for (int kb = 0; kb < nkb; kb++) {
        const int s = kb % NSTAGE, b = kb % NBBUF;
        unsigned char* st = smem + (size_t)s * STAGE_B;
        const int grp = grp_of(kb);
        if (grp != cur_grp) {                      // nxt_* holds exactly this group (fetched during the previous k-block)
            const uint32_t zp = ((nxt_zw >> ((colc & 7) * 4)) & 0xfu) + 1u;
            zs = (0x6400u + zp) * 0x00010001u;
            zf = (0xd400u + (zp << 4)) * 0x00010001u;
            s2 = (uint32_t)nxt_sh * 0x00010001u;
            cur_grp = grp;
        }
        if (kb + 1 < nkb) {
            const int gn = grp_of(kb + 1);
            if (gn != nxt_grp) fetch(gn);
        }
        bar_wait(&full_in[s], (uint32_t)(kb / NSTAGE) & 1u);
        const uint32_t* wq = reinterpret_cast<const uint32_t*>(st + MT * A_BYTES) + (hh * 4) * BN + cn;
        uint32_t w[4];
        #pragma unroll
        for (int i = 0; i < 4; i++) w[i] = wq[i * BN];
        unsigned char* bt = bbuf + (size_t)b * B_BYTES + b_off;
        #pragma unroll
        for (int i = 0; i < 4; i++) {
            // row cn of the K-major SW128 tile, 16-byte chunk r stored at r ^ (cn & 7)
            *reinterpret_cast<uint4*>(bt + (((hh * 4 + i) ^ (cn & 7)) << 4)) = dequant8(w[i], zs, zf, s2);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy stores -> visible to the tensor core
        consumer_sync();                                                  // B tile kb complete (and every wgmma of kb - 2 retired)

        wgmma_fence();
        const uint32_t a_addr = s_u32(st) + (uint32_t)(wg * MT * 64) * 128u;
        const uint32_t b_addr = s_u32(bbuf + (size_t)b * B_BYTES);
        #pragma unroll
        for (int h = 0; h < MT; h++) {
            #pragma unroll
            for (int k = 0; k < BK / 16; k++)
                wgmma_m64n128k16(acc[h], gmma_desc_sw128(a_addr + h * 64 * 128 + k * 32), gmma_desc_sw128(b_addr + k * 32), 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();                                                  // the wgmmas of kb - 1 are done: release their x stage
        if (kb > 0 && (tid & 127) == 0) bar_arrive(&empty[(kb - 1) % NSTAGE]);
    }
    wgmma_wait<0>();

    // ================================ epilogue: accumulator fragment -> out ================================
    // m64n128 fragment: warp w of the warpgroup holds rows 16 w + lane / 4 (+ 8); register 4 j + {0, 1} (+ {2, 3} for row + 8) is
    // columns 8 j + 2 (lane % 4) + {0, 1}
    const int lane = tid & 31, wi = warp & 3;
    #pragma unroll
    for (int h = 0; h < MT; h++) {
        const int r0 = m0 + wg * MT * 64 + h * 64 + wi * 16 + (lane >> 2);
        #pragma unroll
        for (int j = 0; j < BN / 8; j++) {
            const int c = n0 + j * 8 + (lane & 3) * 2;
            if (c >= a.N) continue;                                       // N % 8 == 0: the pair is either in or out
            #pragma unroll
            for (int rr = 0; rr < 2; rr++) {
                const int m = r0 + rr * 8;
                if (m >= a.M) continue;
                half2* p = reinterpret_cast<half2*>(a.out + (size_t)m * a.N + c);
                float f0 = acc[h][4 * j + 2 * rr], f1 = acc[h][4 * j + 2 * rr + 1];
                if (a.no_zero) { const float2 pf = __half22float2(*p); f0 += pf.x; f1 += pf.y; }
                *p = __floats2half2_rn(f0, f1);
            }
        }
    }
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

} // namespace

bool exl_tc_gemm_supported(const exl_q4_matrix* w, int M)
{
    if (M < 1) return false;
    if (w->K % BK != 0 || w->N % 8 != 0) return false;
    if (w->groups > 1) {
        const int gs32 = w->groupsize / 32;
        if (w->groupsize % 32 != 0 || (gs32 & (gs32 - 1)) != 0) return false;
    }
    return true;
}

int exl_tc_gemm_launch(ExlDevice* ds, const half* x, int M, const exl_q4_matrix* w, half* out, bool no_zero, cudaStream_t stream)
{
    if (!exl_tc_gemm_supported(w, M)) return exl_set_err(EXL_ERR_ARG, "tc_gemm: unsupported shape K=%d N=%d groupsize=%d", w->K, w->N, w->groupsize);
    EncodeFn encode = get_encode();
    if (!encode) return exl_set_err(EXL_ERR_CUDA, "tc_gemm: cuTensorMapEncodeTiled unavailable");

    const half* xin = x;
    if (w->x_map) {
        // act-order: gather the columns of x once (column_remap.cu:27-34) so the TMA tile is dense
        const int64_t need = (int64_t)M * w->K;
        half* xm = nullptr;
        if (ds->temp_state && ds->temp_state_numel >= need) xm = ds->temp_state;
        else { int rc = exl_own_scratch(ds, SCR_REMAP, need, &xm); if (rc != EXL_OK) return rc; }
        int rc = exl_column_remap_launch(x, xm, M, w->K, w->x_map, stream);
        if (rc != EXL_OK) return rc;
        xin = xm;
    }

    TcArgs a;
    memset(&a, 0, sizeof(a));
    {
        const cuuint64_t dims[2] = {(cuuint64_t)w->K, (cuuint64_t)M};
        const cuuint64_t strides[1] = {(cuuint64_t)w->K * 2};
        const cuuint32_t box[2] = {BK, BM};
        const cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&a.tmap_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)xin, dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return exl_set_err(EXL_ERR_CUDA, "tc_gemm: tensor map for x failed (%d)", (int)r);
    }
    a.tmap_w = w->tmap_wp;
    a.qz = w->qzeros; a.sc = w->scales; a.out = out;
    a.M = M; a.N = w->N; a.K = w->K; a.groups = w->groups; a.no_zero = no_zero ? 1 : 0;
    int sh = 0; while ((32 << sh) < w->groupsize) sh++;
    a.gs_shift32 = w->groups == 1 ? 30 : sh;

    // tile choice: 256 x 128 (x tiles of two sub-tiles share one dequantised B tile) when that still gives at least half a CTA
    // per SM; smaller problems use 128 x 128 tiles for more CTAs
    const long long t2 = (long long)((M + 2 * BM - 1) / (2 * BM)) * ((w->N + BN - 1) / BN);
    const int mt = (M > BM && t2 >= ds->num_sms / 2) ? 2 : 1;
    const size_t smem = 1024 + (size_t)NSTAGE * (mt * A_BYTES + WQ_BYTES) + (size_t)NBBUF * B_BYTES;
    static int attr_done[EXL_MAX_DEVICES][2] = {};
    void (*kern)(const TcArgs) = mt == 2 ? q4_gemm_tc_kernel<2> : q4_gemm_tc_kernel<1>;
    if (!attr_done[ds->device][mt - 1]) {
        EXL_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done[ds->device][mt - 1] = 1;
    }
    const dim3 grid((unsigned)((w->N + BN - 1) / BN), (unsigned)((M + BM * mt - 1) / (BM * mt)));
    kern<<<grid, TC_THREADS, smem, stream>>>(a);
    EXL_CHECK_LAUNCH("q4_gemm_tc_kernel");
    return EXL_OK;
}
