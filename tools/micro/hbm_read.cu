// hbm_read.cu -- the HBM read rate one CTA per SM reaches with each load mechanism the decode step could use (run through
// hbm_read.py).
//
// The buffer holds `layers` copies of a Llama-7B layer's q4 tensors (q, k, v, o 4096 x 4096; gate, up 4096 x 11008; down
// 11008 x 4096; g128 scales and zeros), 4.2 GB at 40 layers, far more than L2.  One CTA per SM, launched cooperatively.  Lane 0
// of one or four producer warps streams into its part of a shared-memory ring and re-issues a slot as soon as it lands (nothing
// reads the data); with four, each takes every fourth load, as the step's four pipelines do.  Warp 0 lane 0 can run grid
// barriers at the decode step's cadence meanwhile, and then tells the producers to stop through shared memory: a stop flag in
// global memory, read once per load, costs the issue loop an L2 round trip per load and caps the stream at ~2.5 TB/s.  Loads:
//   MODE_BULK  1-D cp.async.bulk of `op` bytes, CTA c takes chunks c, c + G, c + 2G, ... of the buffer;
//   MODE_UNIT  the step kernel's weight units: one 3-D tensor-map op per unit (box {32, 16 * kst, 4}: 16 * kst runs of 512 B at a
//              stride of N * 4 bytes) plus one 2-D op each for the unit's scale and zero rows, over the stream-K range of every
//              phase (QKV, O, GU, DOWN) of every layer;
//   MODE_WIDE  units of four 128-column tiles x 32 k (box {32, 4, 16}: 4 runs of 2 KB), scale and zero rows of 512 columns
//              (1-D bulk copies) with every fourth unit;
//   ld kernel  ld.global.nc.L1::no_allocate.v4 by 16 warps, `unroll` 16-byte loads in flight per thread, discarded.
// Rate = bytes landed / (last landing - first issue) over all CTAs, by %globaltimer.  Every wait is bounded by wall time.
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cstring>
#include <vector>
#include <algorithm>
#include <cuda.h>
#include <cuda_runtime.h>

constexpr int MAX_SLOTS = 16;
constexpr int META = 2048;                       // per slot: scale rows at +0, zero rows at +1280
constexpr unsigned long long WAIT_NS = 4000000000ull;
enum { MODE_BULK = 0, MODE_UNIT = 1, MODE_WIDE = 2 };
enum { ARRIVE_NONE = 0, ARRIVE_RELEASE = 1, ARRIVE_RELAXED = 2 };

struct Mat { const unsigned char* qw; const unsigned char* sc; const unsigned char* zr; int K, N, groups; };
__shared__ Mat s_mat[7];                         // layer 0's tensors; layer l's sit l * layer_bytes further

__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    const unsigned long long t0 = gtime();
    for (unsigned i = 1; !mbar_try(bar, parity); i++)
        if ((i & 1023u) == 0 && gtime() - t0 > WAIT_NS) __trap();
}
__device__ __forceinline__ void bulk(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t pol, bool hint)
{
    if (hint)
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                     :: "r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(pol) : "memory");
    else
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma2(uint32_t dst, const CUtensorMap* m, int c0, int c1, uint32_t bar, uint64_t pol, bool hint)
{
    if (hint)
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3}], [%4], %5;"
                     :: "r"(dst), "l"(m), "r"(c0), "r"(c1), "r"(bar), "l"(pol) : "memory");
    else
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                     :: "r"(dst), "l"(m), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma3(uint32_t dst, const CUtensorMap* m, int c0, int c1, int c2, uint32_t bar, uint64_t pol, bool hint)
{
    if (hint)
        asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3, %4}], [%5], %6;"
                     :: "r"(dst), "l"(m), "r"(c0), "r"(c1), "r"(c2), "r"(bar), "l"(pol) : "memory");
    else
        asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                     :: "r"(dst), "l"(m), "r"(c0), "r"(c1), "r"(c2), "r"(bar) : "memory");
}

struct Args
{
    const unsigned char* buf; long long buf_bytes;
    const Mat* mats; const CUtensorMap* maps;    // [7] (layer 0); maps [layers * 7][3]: weights, scales, zeros
    int layers; long long layer_bytes;
    int mode, op, slots, kst, meta, hint;        // op: bytes per 1-D copy / weight op; kst: K stages (of 128) per MODE_UNIT op
    int arrive, rounds, spin_ns;                 // grid barriers run by thread 0 (rounds > 0: stream until CTA 0's last one)
    int sleep_wait, poll_ns;                     // wait between barriers by __nanosleep instead of a %globaltimer spin; poll back-off
    int prod;                                    // producer warps (1 or 4), each with slots / prod of the ring and every prod-th load
    unsigned long long* bar;
    unsigned* fence_ns; unsigned* barrier_ns;    // [G][rounds]
    unsigned long long* bytes; unsigned long long* t_span;     // [G][4], [G][4][2]
};

// The CTA's walk over the weights, incremental as decode_step_kernel's producers walk it (no division per unit): phase p of layer
// l is matrices [P0[p], P1[p]); the phase's units, tile-major, are cut into G contiguous ranges.
__shared__ int s_upt[7], s_tiles[7];             // units per tile, tiles per matrix
struct Walk
{
    int l, ph, left, m, tile, s;                 // left: units of the CTA's range not yet walked in this phase
    __device__ void start(int cta, int G)
    {
        const int P0[4] = {0, 3, 4, 6}, P1[4] = {3, 4, 6, 7};
        m = P0[ph];
        long long U = 0;
        for (int i = m; i < P1[ph]; i++) U += (long long)s_tiles[i] * s_upt[i];
        int lo = (int)(U * cta / G);
        left = (int)(U * (cta + 1) / G) - lo;
        if (left == 0) return;
        while (lo >= s_tiles[m] * s_upt[m]) { lo -= s_tiles[m] * s_upt[m]; m++; }
        tile = lo / s_upt[m]; s = lo - tile * s_upt[m];
    }
    // next unit: matrix index (layer * 7 + matrix), tile, unit within the tile; false at the end (and wrap == false)
    __device__ bool next(int layers, int cta, int G, bool wrap, int& mi, int& t, int& u)
    {
        while (left == 0) {
            if (++ph == 4) { ph = 0; if (++l == layers) { if (!wrap) return false; l = 0; } }
            start(cta, G);
        }
        mi = l * 7 + m; t = tile; u = s; left--;
        if (++s == s_upt[m]) { s = 0; if (++tile == s_tiles[m]) { tile = 0; m++; } }
        return true;
    }
};

__global__ void __launch_bounds__(160, 1) stream_kernel(const Args a)
{
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    __shared__ __align__(8) unsigned long long full[MAX_SLOTS];
    __shared__ volatile int s_stop;                // set by this CTA's thread 0 after its last barrier
    unsigned char* ring = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int G = (int)gridDim.x, cta = (int)blockIdx.x, tid = threadIdx.x;
    if (tid == 0) {
        for (int i = 0; i < MAX_SLOTS; i++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(&full[i])));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (tid < 7) {
        const Mat m = a.mats[tid];
        s_mat[tid] = m;
        s_upt[tid] = a.mode == MODE_WIDE ? m.K / 32 : (m.K / 128 + a.kst - 1) / a.kst;
        s_tiles[tid] = a.mode == MODE_WIDE ? (m.N + 511) / 512 : m.N / 128;
    }
    if (tid == 0) s_stop = 0;
    __syncthreads();
    const bool barriers = a.rounds > 0;
    const int pw = (tid >> 5) - 1;
    if (pw >= 0 && pw < a.prod && (tid & 31) == 0) {
        const int S = a.slots / a.prod, sb = pw * S;
        uint64_t pol;
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
        const bool hint = a.hint != 0;
        const uint32_t slot_bytes = (uint32_t)a.op + META;
        unsigned long long landed = 0, t_first = gtime(), t_last = t_first;
        uint32_t par[MAX_SLOTS] = {}, tx[MAX_SLOTS] = {};
        long long chunk = cta + (long long)pw * G;
        int k = 0;
        const long long nchunks = a.buf_bytes / a.op;
        Walk w{0, 0, 0, 0, 0, 0};
        if (a.mode != MODE_BULK) w.start(cta, G);
        int s = 0, inflight = 0;
        for (;;) {
            if (inflight == S) {
                mbar_wait(smem_u32(&full[sb + s]), par[s]); par[s] ^= 1u; landed += tx[s]; t_last = gtime(); inflight--;
            }
            if (barriers && s_stop) break;
            const uint32_t dst = smem_u32(ring) + (uint32_t)(sb + s) * slot_bytes, fb = smem_u32(&full[sb + s]);
            uint32_t bytes = 0;
            if (a.mode == MODE_BULK) {
                if (chunk >= nchunks) { if (!barriers) break; chunk -= nchunks; }
                bytes = (uint32_t)a.op;
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(fb), "r"(bytes) : "memory");
                bulk(dst, a.buf + chunk * a.op, bytes, fb, pol, hint);
                chunk += (long long)a.prod * G;
            } else {
                int mi, tile, u;
                bool more = w.next(a.layers, cta, G, barriers, mi, tile, u);
                for (; more && k++ % a.prod != pw;) more = w.next(a.layers, cta, G, barriers, mi, tile, u);
                if (!more) break;
                const Mat& m = s_mat[mi % 7];
                const long long lofs = (long long)(mi / 7) * a.layer_bytes;
                const CUtensorMap* mp = a.maps + 3 * mi;
                if (a.mode == MODE_UNIT) {
                    // bytes the op moves from HBM (the box may reach past K on the last unit of a tile)
                    const int k8 = u * a.kst * 16, rows = min(a.kst * 16, m.K / 8 - k8);
                    const int g0 = u * a.kst, gr = min(a.kst, m.groups - g0);
                    bytes = (uint32_t)rows * 512u + (a.meta ? (uint32_t)gr * 320u : 0u);
                    const uint32_t box = (uint32_t)a.kst * 8192u + (a.meta ? (uint32_t)a.kst * 320u : 0u);
                    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(fb), "r"(box) : "memory");
                    tma3(dst, mp, 0, k8, tile * 4, fb, pol, hint);
                    if (a.meta) {
                        tma2(dst + a.op, mp + 1, tile * 128, g0, fb, pol, hint);
                        tma2(dst + a.op + 1280, mp + 2, tile * 16, g0, fb, pol, hint);
                    }
                } else {
                    const int cols = min(512, m.N - tile * 512);
                    const bool meta = a.meta && (u & 3) == 0;
                    bytes = (uint32_t)cols * 16u + (meta ? (uint32_t)cols * 5u / 2u : 0u);
                    const uint32_t box = 8192u + (meta ? (uint32_t)cols * 5u / 2u : 0u);
                    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(fb), "r"(box) : "memory");
                    tma3(dst, mp, 0, u * 4, tile * 16, fb, pol, hint);
                    if (meta) {
                        const int g = u >> 2;
                        bulk(dst + a.op, m.sc + lofs + ((size_t)g * m.N + tile * 512) * 2, (uint32_t)cols * 2u, fb, pol, hint);
                        bulk(dst + a.op + 1280, m.zr + lofs + ((size_t)g * m.N + tile * 512) / 2, (uint32_t)cols / 2u, fb, pol, hint);
                    }
                }
            }
            tx[s] = bytes; inflight++;
            s = s + 1 == S ? 0 : s + 1;
        }
        for (; inflight > 0; inflight--) {                       // drain, oldest first
            s = (s + S - inflight) % S;
            mbar_wait(smem_u32(&full[sb + s]), par[s]); par[s] ^= 1u; landed += tx[s]; t_last = gtime();
            s = (s + inflight) % S;
        }
        const int o = cta * 4 + pw;
        a.bytes[o] = landed; a.t_span[2 * o] = t_first; a.t_span[2 * o + 1] = t_last;
    } else if (tid == 0 && barriers) {
        // grid barriers as decode_step_kernel's grid_barrier makes them, `spin_ns` apart (ARRIVE_NONE: the wait alone)
        unsigned long long v;
        asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(a.bar) : "memory");
        unsigned long long target = v - v % (unsigned long long)G + (unsigned long long)G;
        for (int r = 0; r < a.rounds; r++) {
            const unsigned long long s0 = gtime();
            if (a.sleep_wait) { while (gtime() - s0 < (unsigned long long)a.spin_ns) __nanosleep(500); }
            else { while (gtime() - s0 < (unsigned long long)a.spin_ns) { } }
            const unsigned long long t0 = gtime();
            if (a.arrive == ARRIVE_NONE) { a.fence_ns[(size_t)cta * a.rounds + r] = a.barrier_ns[(size_t)cta * a.rounds + r] = 0; continue; }
            if (a.arrive == ARRIVE_RELEASE) asm volatile("red.release.gpu.global.add.u64 [%0], 1;" :: "l"(a.bar) : "memory");
            else asm volatile("red.relaxed.gpu.global.add.u64 [%0], 1;" :: "l"(a.bar) : "memory");
            const unsigned long long t1 = gtime();
            unsigned i = 0;
            do {
                if (a.poll_ns && i) __nanosleep(a.poll_ns);
                asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(a.bar) : "memory");
                if ((++i & 1023u) == 0 && gtime() - t0 > WAIT_NS) __trap();
            } while (v < target);
            const unsigned long long t2 = gtime();
            target += (unsigned long long)G;
            a.fence_ns[(size_t)cta * a.rounds + r] = (unsigned)(t1 - t0);
            a.barrier_ns[(size_t)cta * a.rounds + r] = (unsigned)(t2 - t0);
        }
        s_stop = 1;
    }
}

// 16 warps of plain loads: CTA c reads 8 KB chunks c, c + G, ... (one 16-byte load per thread per chunk), UNROLL chunks in flight
template <int UNROLL>
__global__ void __launch_bounds__(512, 1) ld_kernel(const unsigned char* buf, long long nchunks, unsigned long long* bytes,
                                                    unsigned long long* t_span, unsigned* sink)
{
    const int G = (int)gridDim.x, cta = (int)blockIdx.x, tid = threadIdx.x;
    const unsigned long long t0 = gtime();
    uint32_t acc = 0;
    long long c = cta;
    for (; c + (long long)(UNROLL - 1) * G < nchunks; c += (long long)UNROLL * G) {
        uint4 v[UNROLL];
        #pragma unroll
        for (int i = 0; i < UNROLL; i++)
            asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(v[i].x), "=r"(v[i].y), "=r"(v[i].z), "=r"(v[i].w) : "l"(buf + (c + (long long)i * G) * 8192 + tid * 16));
        #pragma unroll
        for (int i = 0; i < UNROLL; i++) acc ^= v[i].x ^ v[i].y ^ v[i].z ^ v[i].w;
    }
    if (acc == 0x9e3779b9u) sink[tid] = acc;                      // never true for the memset pattern; keeps the loads alive
    __syncthreads();
    if (tid == 0) {
        bytes[4 * cta] = (unsigned long long)((c - cta) / G) * 8192ull;
        t_span[8 * cta] = t0; t_span[8 * cta + 1] = gtime();
    }
}

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// the weight / scale / zero maps of exl_encode_weight_tmap (q4_matrix.cu), with the unit box {32, 16 * kst, 4} or, wide, {32, 4, 16}
static void encode(EncodeFn enc, const Mat& m, int kst, bool wide, CUtensorMap* out)
{
    const cuuint64_t d3[3] = {32, (cuuint64_t)(m.K / 8), (cuuint64_t)(m.N / 32)};
    const cuuint64_t s3[2] = {(cuuint64_t)m.N * 4, 128};
    const cuuint32_t b3[3] = {32, wide ? 4u : (cuuint32_t)(16 * kst), wide ? 16u : 4u};
    const cuuint32_t e3[3] = {1, 1, 1};
    CUresult r = enc(&out[0], CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, (void*)m.qw, d3, s3, b3, e3, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    const cuuint64_t dsc[2] = {(cuuint64_t)m.N, (cuuint64_t)m.groups}, ssc[1] = {(cuuint64_t)m.N * 2};
    const cuuint32_t bsc[2] = {128, (cuuint32_t)kst}, estr[2] = {1, 1};
    r = r ? r : enc(&out[1], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)m.sc, dsc, ssc, bsc, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    const cuuint64_t dqz[2] = {(cuuint64_t)(m.N / 8), (cuuint64_t)m.groups}, sqz[1] = {(cuuint64_t)(m.N / 8) * 4};
    const cuuint32_t bqz[2] = {16, (cuuint32_t)kst};
    r = r ? r : enc(&out[2], CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, (void*)m.zr, dqz, sqz, bqz, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { fprintf(stderr, "cuTensorMapEncodeTiled failed (%d) K=%d N=%d\n", (int)r, m.K, m.N); exit(1); }
}

static double pct(std::vector<unsigned> v, double q) { std::sort(v.begin(), v.end()); return v.empty() ? 0.0 : v[(size_t)(q * (v.size() - 1))] / 1e3; }

int main(int argc, char** argv)
{
    const int layers = argc > 1 ? atoi(argv[1]) : 40, reps = argc > 2 ? atoi(argv[2]) : 3;
    const int rounds = argc > 3 ? atoi(argv[3]) : 400, spin_ns = argc > 4 ? atoi(argv[4]) : 10500;
    int dev = 0, sms = 0, coop = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    CK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    if (!coop) { fprintf(stderr, "no cooperative launch\n"); return 1; }
    const int G = sms;
    void* fn = nullptr; cudaDriverEntryPointQueryResult qres;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (qres != cudaDriverEntryPointSuccess || !fn) { fprintf(stderr, "no cuTensorMapEncodeTiled\n"); return 1; }
    const EncodeFn enc = (EncodeFn)fn;

    // the layers' tensors, back to back, each 1 KB aligned
    const int KN[7][2] = {{4096, 4096}, {4096, 4096}, {4096, 4096}, {4096, 4096}, {4096, 11008}, {4096, 11008}, {11008, 4096}};
    auto al = [](size_t x) { return (x + 1023) & ~(size_t)1023; };
    size_t per_layer = 0;
    for (auto& kn : KN) { const size_t g = kn[0] / 128; per_layer += al((size_t)kn[0] * kn[1] / 2) + al(g * kn[1] * 2) + al(g * kn[1] / 2); }
    const size_t total = per_layer * layers;
    unsigned char* buf; CK(cudaMalloc(&buf, total)); CK(cudaMemset(buf, 0x11, total));
    std::vector<Mat> mats; size_t off = 0; unsigned long long w_bytes = 0, meta_bytes = 0;
    for (int l = 0; l < layers; l++)
        for (auto& kn : KN) {
            Mat m; m.K = kn[0]; m.N = kn[1]; m.groups = kn[0] / 128;
            m.qw = buf + off; off += al((size_t)m.K * m.N / 2);
            m.sc = buf + off; off += al((size_t)m.groups * m.N * 2);
            m.zr = buf + off; off += al((size_t)m.groups * m.N / 2);
            mats.push_back(m); w_bytes += (size_t)m.K * m.N / 2; meta_bytes += (size_t)m.groups * m.N * 5 / 2;
        }
    Mat* d_mats; CK(cudaMalloc(&d_mats, mats.size() * sizeof(Mat))); CK(cudaMemcpy(d_mats, mats.data(), mats.size() * sizeof(Mat), cudaMemcpyHostToDevice));
    CUtensorMap* d_maps; CK(cudaMalloc(&d_maps, mats.size() * 3 * sizeof(CUtensorMap)));
    std::vector<CUtensorMap> maps(mats.size() * 3);
    unsigned long long* bar; CK(cudaMalloc(&bar, 256)); CK(cudaMemset(bar, 0, 256));
    unsigned *fns, *bns; CK(cudaMalloc(&fns, (size_t)G * rounds * 4)); CK(cudaMalloc(&bns, (size_t)G * rounds * 4));
    unsigned long long *bytes, *span; CK(cudaMalloc(&bytes, G * 32)); CK(cudaMalloc(&span, G * 64));
    unsigned* sink; CK(cudaMalloc(&sink, 512 * 4));
    CK(cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(ld_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 120 * 1024));
    CK(cudaFuncSetAttribute(ld_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 120 * 1024));

    struct V { const char* variant; const char* what; int mode, op, slots, kst, meta, hint, arrive, unroll, sleep = 0, poll = 0, spin_only = 0, prod = 1; };
    const char* UNIT = "unit: 3-D op {32,16,4} + scale + zero ops, stream-K 7B";
    std::vector<V> vs = {
        {"a", "bulk 8 KB, contiguous chunks", MODE_BULK, 8192, 4, 1, 0, 0, 0, 0},
        {"a", "bulk 8 KB, contiguous chunks", MODE_BULK, 8192, 8, 1, 0, 0, 0, 0},
        {"a", "bulk 8 KB, contiguous chunks", MODE_BULK, 8192, 12, 1, 0, 0, 0, 0},
        {"a", "bulk 8 KB, contiguous chunks", MODE_BULK, 8192, 16, 1, 0, 0, 0, 0},
        {"a", "bulk 8 KB, contiguous chunks, evict-first", MODE_BULK, 8192, 12, 1, 0, 1, 0, 0},
        {"a", "bulk 8 KB, contiguous chunks, 4 producer warps", MODE_BULK, 8192, 12, 1, 0, 0, 0, 0, 0, 0, 0, 4},
        {"b", "bulk 8 KB + grid barriers, red.release arrival", MODE_BULK, 8192, 4, 1, 0, 0, ARRIVE_RELEASE, 0},
        {"b", "bulk 8 KB + grid barriers, red.release arrival", MODE_BULK, 8192, 12, 1, 0, 0, ARRIVE_RELEASE, 0},
        {"b", "bulk 8 KB + grid barriers, red.relaxed arrival", MODE_BULK, 8192, 4, 1, 0, 0, ARRIVE_RELAXED, 0},
        {"b", "bulk 8 KB + grid barriers, red.relaxed arrival", MODE_BULK, 8192, 12, 1, 0, 0, ARRIVE_RELAXED, 0},
        {"b", "bulk 8 KB + the %globaltimer wait alone (no barrier)", MODE_BULK, 8192, 12, 1, 0, 0, ARRIVE_NONE, 0, 0, 0, 1},
        {"b", "bulk 8 KB + grid barriers, red.release, __nanosleep between barriers", MODE_BULK, 8192, 12, 1, 0, 0, ARRIVE_RELEASE, 0, 1, 0},
        {"b", "bulk 8 KB + grid barriers, red.release, __nanosleep between, 100 ns poll back-off", MODE_BULK, 8192, 12, 1, 0, 0, ARRIVE_RELEASE, 0, 1, 100},
        {"c", UNIT, MODE_UNIT, 8192, 4, 1, 1, 0, 0, 0},
        {"c", UNIT, MODE_UNIT, 8192, 8, 1, 1, 0, 0, 0},
        {"c", UNIT, MODE_UNIT, 8192, 12, 1, 1, 0, 0, 0},
        {"c", UNIT, MODE_UNIT, 8192, 16, 1, 1, 0, 0, 0},
        {"c", UNIT, MODE_UNIT, 8192, 12, 1, 1, 1, 0, 0},
        {"c", UNIT, MODE_UNIT, 8192, 16, 1, 1, 1, 0, 0},
        {"c", "unit: 3-D op {32,16,4} only (no scale / zero ops)", MODE_UNIT, 8192, 12, 1, 0, 0, 0, 0},
        {"c", UNIT, MODE_UNIT, 8192, 12, 1, 1, 0, 0, 0, 0, 0, 0, 4},
        {"c", UNIT, MODE_UNIT, 8192, 16, 1, 1, 0, 0, 0, 0, 0, 0, 4},
        {"c", UNIT, MODE_UNIT, 8192, 12, 1, 1, 1, 0, 0, 0, 0, 0, 4},
        {"c", "unit ops + grid barriers, red.release arrival", MODE_UNIT, 8192, 12, 1, 1, 1, ARRIVE_RELEASE, 0, 0, 0, 0, 4},
        {"d", "2 K stages per op: 3-D {32,32,4} + scale + zero", MODE_UNIT, 16384, 6, 2, 1, 0, 0, 0},
        {"d", "2 K stages per op: 3-D {32,32,4} + scale + zero", MODE_UNIT, 16384, 8, 2, 1, 0, 0, 0},
        {"d", "2 K stages per op: 3-D {32,32,4} + scale + zero", MODE_UNIT, 16384, 8, 2, 1, 0, 0, 0, 0, 0, 0, 4},
        {"d", "4 K stages per op: 3-D {32,64,4} + scale + zero", MODE_UNIT, 32768, 3, 4, 1, 0, 0, 0},
        {"d", "4 K stages per op: 3-D {32,64,4} + scale + zero", MODE_UNIT, 32768, 4, 4, 1, 0, 0, 0},
        {"d", "4 K stages per op: 3-D {32,64,4} + scale + zero", MODE_UNIT, 32768, 4, 4, 1, 0, 0, 0, 0, 0, 0, 4},
        {"d", "bulk 16 KB, contiguous chunks", MODE_BULK, 16384, 4, 1, 0, 0, 0, 0},
        {"d", "bulk 16 KB, contiguous chunks", MODE_BULK, 16384, 6, 1, 0, 0, 0, 0},
        {"d", "bulk 16 KB, contiguous chunks", MODE_BULK, 16384, 8, 1, 0, 0, 0, 0},
        {"e", "ld.global.nc.L1::no_allocate.v4, 16 warps", -1, 8192, 0, 1, 0, 0, 0, 4},
        {"e", "ld.global.nc.L1::no_allocate.v4, 16 warps", -1, 8192, 0, 1, 0, 0, 0, 8},
        {"f", "four-tile unit 3-D {32,4,16} (2 KB runs) + scale / zero every 4th", MODE_WIDE, 8192, 12, 1, 1, 0, 0, 0},
        {"f", "four-tile unit 3-D {32,4,16} (2 KB runs) + scale / zero every 4th", MODE_WIDE, 8192, 16, 1, 1, 0, 0, 0},
        {"f", "four-tile unit 3-D {32,4,16} (2 KB runs) + scale / zero every 4th", MODE_WIDE, 8192, 12, 1, 1, 0, 0, 0, 0, 0, 0, 4},
    };
    printf("[");
    for (size_t k = 0; k < vs.size(); k++) {
        const V& v = vs[k];
        if (v.mode == MODE_UNIT || v.mode == MODE_WIDE) {
            for (size_t i = 0; i < mats.size(); i++) encode(enc, mats[i], v.kst, v.mode == MODE_WIDE, &maps[3 * i]);
            CK(cudaMemcpy(d_maps, maps.data(), maps.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice));
        }
        const int rr = v.arrive || v.spin_only ? rounds : 0;
        std::vector<double> gbs, kms; std::vector<unsigned> hf, hb; unsigned long long tot = 0;
        for (int rep = -1; rep < reps; rep++) {                     // rep -1: warm-up
            cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
            CK(cudaEventRecord(e0));
            if (v.mode < 0) {
                const long long nch = (long long)(total / 8192);
                void* kargs[] = {(void*)&buf, (void*)&nch, (void*)&bytes, (void*)&span, (void*)&sink};
                CK(cudaLaunchCooperativeKernel(v.unroll == 4 ? (void*)ld_kernel<4> : (void*)ld_kernel<8>, dim3(G), dim3(512), kargs, 120 * 1024, 0));
            } else {
                Args a{buf, (long long)total, d_mats, d_maps, layers, (long long)per_layer, v.mode, v.op, v.slots, v.kst, v.meta, v.hint,
                       v.arrive, rr, spin_ns, v.sleep, v.poll, v.prod, bar, fns, bns, bytes, span};
                void* kargs[] = {&a};
                const int shm = v.slots * (v.op + META) + 1024;
                CK(cudaLaunchCooperativeKernel((void*)stream_kernel, dim3(G), dim3(32 * (1 + v.prod)), kargs, shm, 0));
            }
            CK(cudaEventRecord(e1));
            CK(cudaDeviceSynchronize());
            float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
            CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1));
            if (rep < 0) continue;
            std::vector<unsigned long long> hby(4 * G), hsp(8 * G);
            CK(cudaMemcpy(hby.data(), bytes, G * 32, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(hsp.data(), span, G * 64, cudaMemcpyDeviceToHost));
            unsigned long long t0 = ~0ull, t1 = 0; tot = 0;
            for (int c = 0; c < 4 * G; c++)
                if (c % 4 < (v.mode < 0 ? 1 : v.prod)) { tot += hby[c]; t0 = std::min(t0, hsp[2 * c]); t1 = std::max(t1, hsp[2 * c + 1]); }
            gbs.push_back(t1 > t0 ? (double)tot / (double)(t1 - t0) : 0.0); kms.push_back(ms);
            if (rr) {
                std::vector<unsigned> f((size_t)G * rr), b((size_t)G * rr);
                CK(cudaMemcpy(f.data(), fns, f.size() * 4, cudaMemcpyDeviceToHost));
                CK(cudaMemcpy(b.data(), bns, b.size() * 4, cudaMemcpyDeviceToHost));
                hf.insert(hf.end(), f.begin(), f.end()); hb.insert(hb.end(), b.begin(), b.end());
            }
        }
        std::vector<double> sg = gbs; std::sort(sg.begin(), sg.end());
        const unsigned long long expect = v.mode < 0 || v.mode == MODE_BULK ? 0ull : w_bytes + (v.meta ? meta_bytes : 0ull);
        printf("%s\n {\"variant\": \"%s\", \"load\": \"%s\", \"op_bytes\": %d, \"ops_in_flight\": %d, \"kb_in_flight\": %d, "
               "\"producer_warps\": %d, \"evict_first\": %d, \"arrival\": \"%s\", \"wait\": \"%s\", \"poll_backoff_ns\": %d, \"hbm_gbs\": %.1f, \"hbm_gbs_min\": %.1f, \"hbm_gbs_max\": %.1f, "
               "\"bytes\": %llu, \"bytes_expected\": %llu, \"kernel_ms\": %.3f, \"fence_us_p50\": %.3f, \"barrier_us_p50\": %.3f, "
               "\"rounds\": %d, \"spin_ns\": %d, \"reps\": %d, \"ctas\": %d}",
               k ? "," : "", v.variant, v.what, v.op, v.mode < 0 ? v.unroll : v.slots,
               v.mode < 0 ? 512 * 16 * v.unroll / 1024 : v.slots * v.op / 1024, v.mode < 0 ? 0 : v.prod, v.hint,
               v.arrive == ARRIVE_RELEASE ? "release" : (v.arrive == ARRIVE_RELAXED ? "relaxed" : "none"),
               rr ? (v.sleep ? "nanosleep" : "globaltimer_spin") : "none", v.poll,
               sg[sg.size() / 2], sg.front(), sg.back(), tot, expect, kms[kms.size() / 2], pct(hf, 0.5), pct(hb, 0.5), rr, rr ? spin_ns : 0,
               reps, G);
        fflush(stdout);
    }
    printf("\n]\n");
    cudaFree(buf); cudaFree(d_mats); cudaFree(d_maps); cudaFree(bar); cudaFree(fns); cudaFree(bns);
    cudaFree(bytes); cudaFree(span); cudaFree(sink);
    return 0;
}
