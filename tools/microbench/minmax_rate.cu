// Issue rate of the min/max flavours a comparator network can be built from (sm_90a): which pipe, how many per clock.
// nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/microbench/minmax_rate.bin tools/microbench/minmax_rate.cu && tools/microbench/minmax_rate.bin
#include <cstdio>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

template <int MODE>
__global__ void __launch_bounds__(256) k(unsigned *out, int iters) {
    unsigned a[8], b[8];
    for (int i = 0; i < 8; ++i) {
        a[i] = threadIdx.x * 2654435761u + i * 40503u;
        b[i] = blockIdx.x * 2246822519u + i * 3266489917u;
    }
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            unsigned lo, hi;
            if (MODE == 0) { lo = min(a[i], b[i]); hi = max(a[i], b[i]); }                       // VIMNMX.U32
            else if (MODE == 1) { lo = __float_as_uint(fminf(__uint_as_float(a[i]), __uint_as_float(b[i])));
                                  hi = __float_as_uint(fmaxf(__uint_as_float(a[i]), __uint_as_float(b[i]))); }   // FMNMX
            else if (MODE == 2) { lo = __vminu2(a[i], b[i]); hi = __vmaxu2(a[i], b[i]); }        // VIMNMX.U16x2
            else if (MODE == 3) { __half2 x = *reinterpret_cast<__half2 *>(&a[i]), y = *reinterpret_cast<__half2 *>(&b[i]);
                                  __half2 l = __hmin2(x, y), h = __hmax2(x, y);
                                  lo = *reinterpret_cast<unsigned *>(&l); hi = *reinterpret_cast<unsigned *>(&h); }   // HMNMX2
            else { lo = __vimin3_u32(a[i], b[i], a[(i + 1) & 7]); hi = __vimax3_u32(a[i], b[i], b[(i + 1) & 7]); }   // VIMNMX3
            a[i] = lo + 1u;   // keep the chain data dependent without adding more than an IADD per pair
            b[i] = hi;
        }
    }
    unsigned s = 0;
    for (int i = 0; i < 8; ++i) s ^= a[i] ^ b[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int MODE>
void run(const char *name) {
    unsigned *d;
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaMalloc(&d, sms * 8 * 256 * sizeof(unsigned));
    const int iters = 20000;
    k<MODE><<<sms * 8, 256>>>(d, 100);
    cudaDeviceSynchronize();
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    cudaEventRecord(a);
    k<MODE><<<sms * 8, 256>>>(d, iters);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    const double ops = (double)sms * 8 * 256 * (double)iters * 8 * 2;   // min + max per pair
    int clk = 0;
    cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    printf("%-14s %8.3f ms  %7.2f Gop/s  = %5.1f min/max per clock per SM (+ 0.5 IADD each) at %d MHz\n", name, ms, ops / ms / 1e6,
           ops / (ms * 1e-3) / sms / (clk * 1e3), clk / 1000);
    cudaFree(d);
}

int main() {
    run<0>("VIMNMX.U32");
    run<1>("FMNMX");
    run<2>("VIMNMX.U16x2");
    run<3>("HMNMX2");
    run<4>("VIMNMX3.U32");
    return 0;
}
