// fence_load.cu -- what a grid-barrier arrival costs while the SM streams HBM (run through fence_load.py).
//
// One CTA per SM, launched cooperatively.  Warp 1 keeps a load on the memory system for the whole kernel:
//   mode 0  bulk copies into shared memory, `kb` KB in flight (kb / 8 stages of 8 KB, each re-issued as soon as it lands);
//   mode 1  the same with 32 KB in flight (four 8 KB stages, as the decode step's four pipelines keep), plus L2 prefetches
//           (cp.async.bulk.prefetch.L2) `ahead` stages in front of those loads, so the loads hit L2.
// CTA c streams 8 KB chunks c, c + G, c + 2G, ... of a buffer much larger than L2.  Thread 0 meanwhile runs `rounds` barriers
// exactly as decode_step_kernel's grid_barrier does (red.release.gpu arrival, ld.acquire.gpu poll), stamping %globaltimer around
// the arrival (fence), around one extra ld.acquire (round trip) and around the whole barrier.  Every wait is bounded by wall time.
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <vector>
#include <algorithm>
#include <cuda_runtime.h>

constexpr int CHUNK = 8192;
constexpr int MAX_STAGES = 16;
constexpr unsigned long long WAIT_NS = 4000000000ull;

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

struct Args
{
    const unsigned char* buf; long long chunks;      // buffer of `chunks` 8 KB chunks
    int mode, stages, ahead, rounds, spin_ns;
    unsigned long long* bar;                         // arrival counter
    volatile int* stop;                              // set by CTA 0 after its last barrier
    unsigned* fence_ns; unsigned* rtt_ns; unsigned* barrier_ns;     // [G][rounds]
    unsigned long long* bytes;                       // [G] bytes landed in shared memory
    unsigned long long* t_span;                      // [G][2] first issue, last landing
};

__global__ void __launch_bounds__(64, 1) fence_load(const Args a)
{
    extern __shared__ __align__(128) unsigned char ring[];
    __shared__ __align__(8) unsigned long long full[MAX_STAGES];
    const int G = (int)gridDim.x, cta = (int)blockIdx.x, tid = threadIdx.x;
    if (tid == 0) {
        for (int i = 0; i < MAX_STAGES; i++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(&full[i])));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 32) {
        // ---------------- producer ----------------
        unsigned long long landed = 0, t_first = gtime(), t_last = t_first;
        long long next = cta, pf = cta;
        uint32_t par[MAX_STAGES] = {};
        auto chunk = [&](long long i) { return a.buf + (size_t)(i % a.chunks) * CHUNK; };
        auto issue = [&](int s) {
            const uint32_t fb = smem_u32(&full[s]);
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(fb), "r"(CHUNK) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         :: "r"(smem_u32(ring) + (uint32_t)s * CHUNK), "l"(chunk(next)), "r"(CHUNK), "r"(fb) : "memory");
            next += G;
            if (a.mode == 1) { asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(chunk(pf)), "r"(CHUNK) : "memory"); pf += G; }
        };
        if (a.stages > 0) {
            if (a.mode == 1)
                for (int k = 0; k < a.ahead; k++) { asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(chunk(pf)), "r"(CHUNK) : "memory"); pf += G; }
            for (int s = 0; s < a.stages; s++) issue(s);
            for (int s = 0; !*a.stop; s = (s + 1 == a.stages ? 0 : s + 1)) {
                mbar_wait(smem_u32(&full[s]), par[s]); par[s] ^= 1u;
                landed += CHUNK; t_last = gtime();
                issue(s);
            }
            for (int k = 0; k < a.stages; k++) {                   // drain: every stage has one copy outstanding
                const int s = k;
                mbar_wait(smem_u32(&full[s]), par[s]); par[s] ^= 1u;
                landed += CHUNK; t_last = gtime();
            }
        }
        a.bytes[cta] = landed; a.t_span[2 * cta] = t_first; a.t_span[2 * cta + 1] = t_last;
    } else if (tid == 0) {
        // ---------------- thread 0: grid barriers under that load ----------------
        unsigned long long v;
        asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(a.bar) : "memory");
        unsigned long long target = v - v % (unsigned long long)G + (unsigned long long)G;
        for (int r = 0; r < a.rounds; r++) {
            const unsigned long long s0 = gtime();
            while (gtime() - s0 < (unsigned long long)a.spin_ns) { }       // let the load settle between barriers
            const unsigned long long t0 = gtime();
            asm volatile("red.release.gpu.global.add.u64 [%0], 1;" :: "l"(a.bar) : "memory");
            const unsigned long long t1 = gtime();
            asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(a.bar) : "memory");
            const unsigned long long t2 = gtime();
            unsigned i = 0;
            while (v < target) {
                asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(a.bar) : "memory");
                if ((++i & 1023u) == 0 && gtime() - t0 > WAIT_NS) __trap();
            }
            const unsigned long long t3 = gtime();
            target += (unsigned long long)G;
            a.fence_ns[(size_t)cta * a.rounds + r] = (unsigned)(t1 - t0);
            a.rtt_ns[(size_t)cta * a.rounds + r] = (unsigned)(t2 - t1);
            a.barrier_ns[(size_t)cta * a.rounds + r] = (unsigned)(t3 - t0);
        }
        *a.stop = 1;
    }
}

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

static double pct(std::vector<unsigned>& v, double q) { std::sort(v.begin(), v.end()); return v[(size_t)(q * (v.size() - 1))] / 1e3; }

int main(int argc, char** argv)
{
    const long long buf_mb = argc > 1 ? atoll(argv[1]) : 2048;
    const int rounds = argc > 2 ? atoi(argv[2]) : 2000, spin_ns = argc > 3 ? atoi(argv[3]) : 3000;
    int dev = 0, sms = 0, coop = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    CK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    if (!coop) { fprintf(stderr, "no cooperative launch\n"); return 1; }
    CK(cudaFuncSetAttribute(fence_load, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_STAGES * CHUNK));
    const int G = sms;
    unsigned char* buf; CK(cudaMalloc(&buf, (size_t)buf_mb << 20)); CK(cudaMemset(buf, 1, (size_t)buf_mb << 20));
    unsigned long long* bar; CK(cudaMalloc(&bar, 256)); CK(cudaMemset(bar, 0, 256));
    int* stop; CK(cudaMalloc(&stop, 4));
    unsigned *f, *rt, *bn; CK(cudaMalloc(&f, (size_t)G * rounds * 4)); CK(cudaMalloc(&rt, (size_t)G * rounds * 4)); CK(cudaMalloc(&bn, (size_t)G * rounds * 4));
    unsigned long long *bytes, *span; CK(cudaMalloc(&bytes, G * 8)); CK(cudaMalloc(&span, G * 16));
    struct Setting { const char* kind; int mode, stages, ahead; double param; };
    std::vector<Setting> settings = {{"bulk_kb", 0, 0, 0, 0}, {"bulk_kb", 0, 4, 0, 32}, {"bulk_kb", 0, 8, 0, 64}, {"bulk_kb", 0, 16, 0, 128}};
    for (int mb : {4, 8, 16, 32}) {
        const int ahead = (int)(((long long)mb << 20) / ((long long)G * CHUNK));           // chunks per CTA for a chip-wide lookahead of mb
        settings.push_back({"prefetch_mb", 1, 4, ahead, (double)mb});
    }
    printf("[");
    for (size_t k = 0; k < settings.size(); k++) {
        const Setting& s = settings[k];
        for (int warm = 0; warm < 2; warm++) {
            CK(cudaMemset(stop, 0, 4));
            Args a{buf, ((long long)buf_mb << 20) / CHUNK, s.mode, s.stages, s.ahead, rounds, spin_ns, bar, stop, f, rt, bn, bytes, span};
            void* kargs[] = {&a};
            cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
            CK(cudaEventRecord(e0));
            CK(cudaLaunchCooperativeKernel((void*)fence_load, dim3(G), dim3(64), kargs, MAX_STAGES * CHUNK, 0));
            CK(cudaEventRecord(e1));
            CK(cudaDeviceSynchronize());
            float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
            if (!warm) continue;
            std::vector<unsigned> hf((size_t)G * rounds), hr((size_t)G * rounds), hb((size_t)G * rounds);
            std::vector<unsigned long long> hby(G), hsp(2 * G);
            CK(cudaMemcpy(hf.data(), f, hf.size() * 4, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(hr.data(), rt, hr.size() * 4, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(hb.data(), bn, hb.size() * 4, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(hby.data(), bytes, G * 8, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(hsp.data(), span, G * 16, cudaMemcpyDeviceToHost));
            unsigned long long tot = 0, t0 = ~0ull, t1 = 0;
            for (int c = 0; c < G; c++) { tot += hby[c]; t0 = std::min(t0, hsp[2 * c]); t1 = std::max(t1, hsp[2 * c + 1]); }
            const double gbs = t1 > t0 ? (double)tot / (double)(t1 - t0) : 0.0;              // bytes per ns = GB/s
            printf("%s\n {\"load\": \"%s\", \"value\": %g, \"stages_in_flight\": %d, \"ahead_chunks_per_cta\": %d, \"chip_lookahead_mb\": %.2f, "
                   "\"fence_us_p50\": %.3f, \"fence_us_p90\": %.3f, \"rtt_us_p50\": %.3f, \"rtt_us_p90\": %.3f, \"barrier_us_p50\": %.3f, "
                   "\"hbm_gbs\": %.1f, \"bytes\": %llu, \"kernel_ms\": %.3f, \"ctas\": %d, \"rounds\": %d, \"spin_ns\": %d}",
                   k ? "," : "", s.kind, s.param, s.stages, s.ahead, (double)s.ahead * G * CHUNK / (1 << 20),
                   pct(hf, 0.5), pct(hf, 0.9), pct(hr, 0.5), pct(hr, 0.9), pct(hb, 0.5), gbs, tot, ms, G, rounds, spin_ns);
            CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1));
        }
    }
    printf("\n]\n");
    cudaFree(buf); cudaFree(bar); cudaFree(stop); cudaFree(f); cudaFree(rt); cudaFree(bn); cudaFree(bytes); cudaFree(span);
    return 0;
}
