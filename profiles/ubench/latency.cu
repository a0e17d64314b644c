// Dependent-issue latency of a few SASS instructions on the device this runs on (profiling aid).
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -fmad=false -o latency latency.cu
#include <cstdio>
#include <cuda_runtime.h>

template <int OP>
__global__ void chain(double* out, double a, double b, int n, long long* cycles) {
    double x = a;
    float xf = (float)a, bf = (float)b;
    unsigned xi = (unsigned)a;
    long long t0 = clock64();
#pragma unroll 1
    for (int i = 0; i < n; ++i) {
#pragma unroll
        for (int u = 0; u < 32; ++u) {
            if (OP == 0) x = x + b;
            if (OP == 1) x = x * b;
            if (OP == 2) x = fma(x, b, a);
            if (OP == 3) xf = xf + bf;
            if (OP == 4) xf = fmaf(xf, bf, bf);
            if (OP == 5) xi = xi * 3u + 7u;
            if (OP == 6) x = (double)(float)x + b;            // F2F round trip + DADD
            if (OP == 7) x = __drcp_rn(x) + b;
            if (OP == 8) x = sqrt(x) + b;
            if (OP == 9) xf = __shfl_sync(0xffffffffu, xf, 1) + bf;
        }
    }
    long long t1 = clock64();
    if (threadIdx.x == 0) { out[0] = x + xf + xi; cycles[0] = t1 - t0; }
}

int main() {
    double* out; long long* cyc;
    cudaMalloc(&out, 8); cudaMalloc(&cyc, 8);
    const char* names[] = {"DADD", "DMUL", "DFMA", "FADD", "FFMA", "IMAD", "F2F.F32.F64+F2F.F64.F32+DADD", "drcp_rn+DADD", "dsqrt+DADD", "SHFL+FADD"};
    const int n = 256;
    for (int warps = 1; warps <= 16; warps *= 4) {
        printf("-- %d warp(s) per block, 1 block\n", warps);
        for (int op = 0; op < 10; ++op) {
            long long h = 0;
            for (int rep = 0; rep < 2; ++rep) {
                switch (op) {
                    case 0: chain<0><<<1, 32 * warps>>>(out, 1.0, 1e-9, n, cyc); break;
                    case 1: chain<1><<<1, 32 * warps>>>(out, 1.0, 1.0000001, n, cyc); break;
                    case 2: chain<2><<<1, 32 * warps>>>(out, 1.0, 0.5, n, cyc); break;
                    case 3: chain<3><<<1, 32 * warps>>>(out, 1.0, 1e-9, n, cyc); break;
                    case 4: chain<4><<<1, 32 * warps>>>(out, 1.0, 0.5, n, cyc); break;
                    case 5: chain<5><<<1, 32 * warps>>>(out, 1.0, 0.5, n, cyc); break;
                    case 6: chain<6><<<1, 32 * warps>>>(out, 1.0, 1e-3, n, cyc); break;
                    case 7: chain<7><<<1, 32 * warps>>>(out, 1.5, 0.5, n, cyc); break;
                    case 8: chain<8><<<1, 32 * warps>>>(out, 1.5, 0.5, n, cyc); break;
                    case 9: chain<9><<<1, 32 * warps>>>(out, 1.5, 0.5, n, cyc); break;
                }
                cudaDeviceSynchronize();
                cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
            }
            printf("%-32s %.1f cycles/op\n", names[op], (double)h / (n * 32));
        }
    }
    return 0;
}
