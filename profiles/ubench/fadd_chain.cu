// Microbenchmark: the floor of an exact sequential float sum on sm_90a.
//   (a) a pure register chain of dependent FADDs (issue-to-use latency),
//   (b) the leader's loop: 16 addends per step from shared memory, the next 16 prefetched (flb_kernels.cuh, error team),
//   (c) the same with 32 addends per step.
// One thread; cycles from clock64().  Build:  nvcc -O3 -arch=sm_90a -fmad=false -o fadd_chain fadd_chain.cu
#include <cstdio>
#include <cuda_runtime.h>

__global__ void k_pure(float* out, long long* cyc, float a, int n) {
    float e = a;
    const long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < n; ++i) e = e + a;
    const long long t1 = clock64();
    out[0] = e;
    cyc[0] = t1 - t0;
}

__global__ void k_smem16(const float* in, float* out, long long* cyc, int n) {
    extern __shared__ __align__(16) float s[];
    for (int i = threadIdx.x; i < n; i += blockDim.x) s[i] = in[i];
    __syncthreads();
    if (threadIdx.x != 0) return;
    const float4* s4 = reinterpret_cast<const float4*>(s);
    float e = 0.f;
    const long long t0 = clock64();
    float4 n0 = s4[0], n1 = s4[1], n2 = s4[2], n3 = s4[3];
    int i = 0;
    for (; i + 16 <= n; i += 16) {
        const float4 c0 = n0, c1 = n1, c2 = n2, c3 = n3;
        const int q = min((i >> 2) + 4, (n >> 2) - 4);
        n0 = s4[q]; n1 = s4[q + 1]; n2 = s4[q + 2]; n3 = s4[q + 3];
        e = e + c0.x; e = e + c0.y; e = e + c0.z; e = e + c0.w;
        e = e + c1.x; e = e + c1.y; e = e + c1.z; e = e + c1.w;
        e = e + c2.x; e = e + c2.y; e = e + c2.z; e = e + c2.w;
        e = e + c3.x; e = e + c3.y; e = e + c3.z; e = e + c3.w;
    }
    const long long t1 = clock64();
    out[0] = e;
    cyc[0] = t1 - t0;
}

__global__ void k_smem32(const float* in, float* out, long long* cyc, int n) {
    extern __shared__ __align__(16) float s[];
    for (int i = threadIdx.x; i < n; i += blockDim.x) s[i] = in[i];
    __syncthreads();
    if (threadIdx.x != 0) return;
    const float4* s4 = reinterpret_cast<const float4*>(s);
    float e = 0.f;
    const long long t0 = clock64();
    float4 nx[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) nx[k] = s4[k];
    int i = 0;
    for (; i + 32 <= n; i += 32) {
        float4 c[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) c[k] = nx[k];
        const int q = min((i >> 2) + 8, (n >> 2) - 8);
#pragma unroll
        for (int k = 0; k < 8; ++k) nx[k] = s4[q + k];
#pragma unroll
        for (int k = 0; k < 8; ++k) { e = e + c[k].x; e = e + c[k].y; e = e + c[k].z; e = e + c[k].w; }
    }
    const long long t1 = clock64();
    out[0] = e;
    cyc[0] = t1 - t0;
}

int main() {
    const int n = 8192;
    float *in, *out;
    long long* cyc;
    cudaMalloc(&in, n * 4); cudaMalloc(&out, 4); cudaMalloc(&cyc, 8);
    float* h = new float[n];
    for (int i = 0; i < n; ++i) h[i] = 1.0f + (i % 7) * 0.125f;
    cudaMemcpy(in, h, n * 4, cudaMemcpyHostToDevice);
    long long c;
    for (int rep = 0; rep < 2; ++rep) {
        k_pure<<<1, 1>>>(out, cyc, 1.5f, n); cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
        if (rep) printf("pure register FADD chain      : %.2f cycles / add\n", (double)c / n);
        k_smem16<<<1, 128, n * 4>>>(in, out, cyc, n); cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
        if (rep) printf("smem, 16 per step, prefetched : %.2f cycles / add\n", (double)c / n);
        k_smem32<<<1, 128, n * 4>>>(in, out, cyc, n); cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
        if (rep) printf("smem, 32 per step, prefetched : %.2f cycles / add\n", (double)c / n);
    }
    int clk = 0;
    cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    printf("SM clock (attr) %d kHz; error: %s\n", clk, cudaGetErrorString(cudaGetLastError()));
    return 0;
}
