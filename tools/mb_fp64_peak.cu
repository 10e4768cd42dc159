// Microbenchmark: fp64 peak (sm_90a) for DFMA and the mma.sync f64 shapes.
// Measured denominator for the Cholesky trailing-update roofline.
// Usage: ./mb_fp64_peak [iters]
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

template <int NACC>
__global__ void k_dfma(double* out, int iters, double a, double b) {
    double acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; i++) acc[i] = threadIdx.x + i;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < NACC; i++) acc[i] = fma(acc[i], a, b);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < NACC; i++) s += acc[i];
    if (s == 123.456) out[0] = s;
}

__device__ __forceinline__ void mma884(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__device__ __forceinline__ void mma1684(double* c, const double* a, double b) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b));
}
__device__ __forceinline__ void mma1688(double* c, const double* a, const double* b) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
__device__ __forceinline__ void mma16816(double* c, const double* a, const double* b) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                   "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

template <int NACC>
__global__ void k_mma884(double* out, int iters) {
    double c[NACC][2];
#pragma unroll
    for (int i = 0; i < NACC; i++) { c[i][0] = i; c[i][1] = threadIdx.x; }
    double a = threadIdx.x * 1e-3, b = 1.0 - threadIdx.x * 1e-3;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < NACC; i++) mma884(c[i][0], c[i][1], a, b);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < NACC; i++) s += c[i][0] + c[i][1];
    if (s == 123.456) out[0] = s;
}
template <int NACC, int SHAPE>
__global__ void k_mma16(double* out, int iters) {
    double c[NACC][4];
#pragma unroll
    for (int i = 0; i < NACC; i++) { c[i][0] = i; c[i][1] = threadIdx.x; c[i][2] = 1; c[i][3] = 2; }
    double a[8], b[4];
#pragma unroll
    for (int i = 0; i < 8; i++) a[i] = threadIdx.x * 1e-3 + i;
#pragma unroll
    for (int i = 0; i < 4; i++) b[i] = 1.0 - threadIdx.x * 1e-3 * i;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < NACC; i++) {
            if (SHAPE == 4) mma1684(c[i], a, b[0]);
            if (SHAPE == 8) mma1688(c[i], a, b);
            if (SHAPE == 16) mma16816(c[i], a, b);
        }
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < NACC; i++) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
    if (s == 123.456) out[0] = s;
}

template <typename F>
double time_ms(F launch) {
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    launch(); CK(cudaGetLastError()); CK(cudaDeviceSynchronize());   // a failed launch (too many registers x 1024 threads) must not be timed
    float best = 1e30f;
    for (int r = 0; r < 3; r++) {
        CK(cudaEventRecord(e0)); launch(); CK(cudaGetLastError()); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
    }
    return best;
}

int main(int argc, char** argv) {
    int iters = argc > 1 ? atoi(argv[1]) : 20000;
    cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
    int sms = p.multiProcessorCount;
    printf("device %s, %d SMs\n", p.name, sms);
    double* out; CK(cudaMalloc(&out, 8));
    for (int warps = 4; warps <= 32; warps *= 2) {
        int threads = warps * 32, blocks = sms * (warps >= 32 ? 1 : 2);
        double totw = (double)blocks * warps;
        double ms;
        ms = time_ms([&] { k_dfma<8><<<blocks, threads>>>(out, iters, 1.0000001, 1e-9); });
        printf("{\"kind\":\"dfma\",\"warps_per_cta\":%d,\"ctas\":%d,\"tflops\":%.2f}\n", warps, blocks,
               totw * 32 * 8 * 2.0 * iters / (ms * 1e-3) / 1e12);
        ms = time_ms([&] { k_mma884<8><<<blocks, threads>>>(out, iters); });
        printf("{\"kind\":\"dmma_m8n8k4\",\"warps_per_cta\":%d,\"ctas\":%d,\"tflops\":%.2f}\n", warps, blocks,
               totw * 8 * 512.0 * iters / (ms * 1e-3) / 1e12);
        ms = time_ms([&] { k_mma16<8, 4><<<blocks, threads>>>(out, iters); });
        printf("{\"kind\":\"dmma_m16n8k4\",\"warps_per_cta\":%d,\"ctas\":%d,\"tflops\":%.2f}\n", warps, blocks,
               totw * 8 * 1024.0 * iters / (ms * 1e-3) / 1e12);
        ms = time_ms([&] { k_mma16<8, 8><<<blocks, threads>>>(out, iters); });
        printf("{\"kind\":\"dmma_m16n8k8\",\"warps_per_cta\":%d,\"ctas\":%d,\"tflops\":%.2f}\n", warps, blocks,
               totw * 8 * 2048.0 * iters / (ms * 1e-3) / 1e12);
        ms = time_ms([&] { k_mma16<8, 16><<<blocks, threads>>>(out, iters); });
        printf("{\"kind\":\"dmma_m16n8k16\",\"warps_per_cta\":%d,\"ctas\":%d,\"tflops\":%.2f}\n", warps, blocks,
               totw * 8 * 4096.0 * iters / (ms * 1e-3) / 1e12);
    }
    return 0;
}
