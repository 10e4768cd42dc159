// Microbenchmark of the DMMA inner loop fed from shared memory (no global traffic): isolates
// whether the LDS.64 fragment loads + DMMA.8x8x4 issue pattern of gemm_nt.cu can reach the
// DMMA peak that tools/mb_fp64_peak measures.  Variants: warp tile shape, CTAs/SM, fragment reuse.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

__device__ __forceinline__ void dmma(double (&c)[2], double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}

// RF x CF fragments per k4 step (warp tile = RF*8 rows x CF*8 cols), KC k-slab, smem [k][row]
template <int RF, int CF, int WARPS, int LDSA, int LDSB>
__global__ void __launch_bounds__(WARPS * 32) k_loop(double* out, int iters) {
    extern __shared__ double sm[];
    constexpr int KC = 16;
    double* sA = sm;
    double* sB = sm + KC * LDSA;
    for (int i = threadIdx.x; i < KC * (LDSA + LDSB); i += blockDim.x) sm[i] = 1e-3 * (i % 97);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gid = lane >> 2, tig = lane & 3;
    const int wr = warp % 4, wc = warp / 4;
    double acc[CF][RF][2];
#pragma unroll
    for (int j = 0; j < CF; j++)
#pragma unroll
        for (int i = 0; i < RF; i++) acc[j][i][0] = acc[j][i][1] = 0.0;
    const double* a = sA + (wr * RF * 8) % 128 + gid;
    const double* b = sB + (wc * CF * 8) % 64 + gid;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int k4 = 0; k4 < KC / 4; k4++) {
            double rf[RF], cf[CF];
#pragma unroll
            for (int i = 0; i < RF; i++) rf[i] = a[(k4 * 4 + tig) * LDSA + i * 8];
#pragma unroll
            for (int j = 0; j < CF; j++) cf[j] = b[(k4 * 4 + tig) * LDSB + j * 8];
#pragma unroll
            for (int j = 0; j < CF; j++)
#pragma unroll
                for (int i = 0; i < RF; i++) dmma(acc[j][i], cf[j], rf[i]);
        }
    }
    double s = 0;
#pragma unroll
    for (int j = 0; j < CF; j++)
#pragma unroll
        for (int i = 0; i < RF; i++) s += acc[j][i][0] + acc[j][i][1];
    if (s == 123.456) out[0] = s;
}

template <int RF, int CF, int WARPS, int LDSA, int LDSB>
void run(const char* name, int ctas_per_sm, int sms, double* out, int iters) {
    auto kern = k_loop<RF, CF, WARPS, LDSA, LDSB>;
    size_t smem = 16 * (LDSA + LDSB) * 8;
    // pad dynamic smem so that exactly ctas_per_sm CTAs fit
    size_t want = (ctas_per_sm == 1) ? 120 * 1024 : (ctas_per_sm == 2 ? 100 * 1024 : 60 * 1024);
    if (want > smem) smem = want;
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int blocks = sms * ctas_per_sm;
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    kern<<<blocks, WARPS * 32, smem>>>(out, iters); CK(cudaDeviceSynchronize());
    float best = 1e30f;
    for (int r = 0; r < 3; r++) {
        CK(cudaEventRecord(e0)); kern<<<blocks, WARPS * 32, smem>>>(out, iters); CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1)); float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
    }
    double flops = (double)blocks * WARPS * iters * 4.0 * RF * CF * 512.0;
    printf("{\"variant\":\"%s\",\"rf\":%d,\"cf\":%d,\"warps\":%d,\"ctas_per_sm\":%d,\"tflops\":%.2f}\n", name, RF, CF, WARPS,
           ctas_per_sm, flops / (best * 1e-3) / 1e12);
}

int main(int argc, char** argv) {
    int iters = argc > 1 ? atoi(argv[1]) : 4000;
    cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
    int sms = p.multiProcessorCount;
    double* out; CK(cudaMalloc(&out, 8));
    run<4, 4, 8, 132, 68>("32x32 warp tile, 8 warps, 2 CTA/SM (current)", 2, sms, out, iters);
    run<4, 4, 8, 132, 68>("32x32 warp tile, 8 warps, 1 CTA/SM", 1, sms, out, iters);
    run<4, 4, 16, 132, 132>("32x32 warp tile, 16 warps, 1 CTA/SM", 1, sms, out, iters);
    run<8, 4, 8, 132, 132>("64x32 warp tile, 8 warps, 1 CTA/SM", 1, sms, out, iters);
    run<8, 4, 4, 132, 132>("64x32 warp tile, 4 warps, 2 CTA/SM", 2, sms, out, iters);
    run<4, 8, 8, 132, 132>("32x64 warp tile, 8 warps, 1 CTA/SM", 1, sms, out, iters);
    run<8, 8, 4, 132, 132>("64x64 warp tile, 4 warps, 1 CTA/SM", 1, sms, out, iters);
    run<2, 2, 8, 132, 68>("16x16 warp tile, 8 warps, 2 CTA/SM", 2, sms, out, iters);
    run<4, 2, 8, 132, 68>("32x16 warp tile, 8 warps, 2 CTA/SM", 2, sms, out, iters);
    return 0;
}
