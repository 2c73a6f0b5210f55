// micro-benchmark: legacy mma.sync throughput/latency on sm_90a: HMMA m16n8k16 f16->f32 vs IMMA m16n8k32 u8.s8->s32
#include <cstdio>
#include <cuda_runtime.h>
#include <cstdint>
template <int MODE, int ILP>
__global__ void k(int iters, int* out, long long* cyc)
{
    int c[ILP][4]; float f[ILP][4];
    #pragma unroll
    for (int i = 0; i < ILP; i++) for (int j = 0; j < 4; j++) { c[i][j] = 0; f[i][j] = 0.f; }
    uint32_t a0 = threadIdx.x, a1 = a0 * 3, a2 = a0 * 5, a3 = a0 * 7, b0 = a0 * 11, b1 = a0 * 13;
    long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
        #pragma unroll
        for (int i = 0; i < ILP; i++) {
            if (MODE == 0)
                asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                             : "+f"(f[i][0]), "+f"(f[i][1]), "+f"(f[i][2]), "+f"(f[i][3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
            else
                asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                             : "+r"(c[i][0]), "+r"(c[i][1]), "+r"(c[i][2]), "+r"(c[i][3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
        }
    }
    long long t1 = clock64();
    int s = 0; float fs = 0;
    #pragma unroll
    for (int i = 0; i < ILP; i++) for (int j = 0; j < 4; j++) { s += c[i][j]; fs += f[i][j]; }
    out[blockIdx.x * blockDim.x + threadIdx.x] = s + (int)fs;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
template <int MODE, int ILP>
void run(const char* name, int warps)
{
    int* out; long long* cyc; cudaMalloc(&out, 132 * 1024 * 4); cudaMalloc(&cyc, 8);
    int iters = 4096;
    k<MODE, ILP><<<132, warps * 32>>>(iters, out, cyc);
    cudaDeviceSynchronize();
    k<MODE, ILP><<<132, warps * 32>>>(iters, out, cyc);
    cudaDeviceSynchronize();
    long long h; cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
    double per = (double)h / (iters * ILP);
    printf("%s warps/SM=%2d ILP=%d: %.2f cycles per mma per warp  -> %.3f mma/cycle/SM\n", name, warps, ILP, per, warps / per);
    cudaFree(out); cudaFree(cyc);
}
int main()
{
    run<0, 1>("HMMA.16816.F32 ", 1); run<0, 2>("HMMA.16816.F32 ", 1); run<0, 4>("HMMA.16816.F32 ", 4); run<0, 4>("HMMA.16816.F32 ", 16);
    run<1, 1>("IMMA.16832.U8S8", 1); run<1, 2>("IMMA.16832.U8S8", 1); run<1, 4>("IMMA.16832.U8S8", 4); run<1, 4>("IMMA.16832.U8S8", 16);
    return 0;
}
