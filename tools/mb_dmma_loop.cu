// Microbenchmark of the DMMA inner loop fed from shared memory (no global traffic): isolates
// whether the LDS.64 fragment loads + DMMA issue pattern of gemm_nt.cu can reach the
// DMMA peak that tools/mb_fp64_peak measures.  Variants: MMA shape, warp tile shape, CTAs/SM,
// fragment reuse.  Every line reports the CTAs per SM the occupancy calculator grants the variant
// and its registers / local-memory bytes, so a variant that does not fit its label is visible.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

__device__ __forceinline__ void dmma(double (&c)[2], double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}
// sm_90 shapes: A fragment a[2g + h] = (m = gid + 8h, k = tig + 4g), B fragment b[g] = (k = tig + 4g, n = gid)
__device__ __forceinline__ void dmma16(double (&c)[4], const double (&a)[2], const double (&b)[1]) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
}
__device__ __forceinline__ void dmma16(double (&c)[4], const double (&a)[4], const double (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
__device__ __forceinline__ void dmma16(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                   "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// Each iteration reads the next of RING k-slabs, as the kernel reads a new ring stage per k-chunk (a
// single slab would let the compiler hoist the loop-invariant fragment loads into registers).
constexpr int RING = 2;

// RF x CF fragments per k4 step (warp tile = RF*8 rows x CF*8 cols), KC k-slab, smem [k][row]
template <int RF, int CF, int WARPS, int LDSA, int LDSB>
__global__ void __launch_bounds__(WARPS * 32) k_loop(double* out, int iters) {
    extern __shared__ double sm[];
    constexpr int KC = 16;
    double* sA = sm;
    double* sB = sm + RING * KC * LDSA;
    for (int i = threadIdx.x; i < RING * KC * (LDSA + LDSB); i += blockDim.x) sm[i] = 1e-3 * (i % 97);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gid = lane >> 2, tig = lane & 3;
    const int wr = warp % 4, wc = warp / 4;
    double acc[CF][RF][2];
#pragma unroll
    for (int j = 0; j < CF; j++)
#pragma unroll
        for (int i = 0; i < RF; i++) acc[j][i][0] = acc[j][i][1] = 0.0;
    const double* a0 = sA + (wr * RF * 8) % 128 + gid;
    const double* b0 = sB + (wc * CF * 8) % 64 + gid;
    for (int it = 0; it < iters; it++) {
        const double* a = a0 + (it & (RING - 1)) * KC * LDSA;
        const double* b = b0 + (it & (RING - 1)) * KC * LDSB;
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

// The 32x32 warp tile of gemm_nt.cu on an m16n8k{KS} shape, fed the way the kernel feeds it: the MMA is
// issued "transposed" (m <-> C columns from sB, n <-> C rows from sA); one 16-column MMA A operand is the
// two 8-column fragments 2jj, 2jj+1 of the m8n8k4 loop.  8 MMAs per KS-deep step.  MAXREG = 112 is the
// cap gemm_nt.cu runs under (2 CTAs of 288 threads per SM); 255 leaves ptxas free (1 CTA per SM).
template <int KS, int MAXREG, int WARPS, int LDSA, int LDSB>
__global__ void __maxnreg__(MAXREG) k_loop16(double* out, int iters) {
    extern __shared__ double sm[];
    constexpr int KC = 16, G = KS / 4;
    double* sA = sm;
    double* sB = sm + RING * KC * LDSA;
    for (int i = threadIdx.x; i < RING * KC * (LDSA + LDSB); i += blockDim.x) sm[i] = 1e-3 * (i % 97);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gid = lane >> 2, tig = lane & 3;
    const int wr = warp % 4, wc = warp / 4;
    double acc[2][4][4];
#pragma unroll
    for (int jj = 0; jj < 2; jj++)
#pragma unroll
        for (int i = 0; i < 4; i++) acc[jj][i][0] = acc[jj][i][1] = acc[jj][i][2] = acc[jj][i][3] = 0.0;
    const double* a0 = sA + (wr * 32) % 128 + gid + tig * LDSA;
    const double* b0 = sB + (wc * 32) % 64 + gid + tig * LDSB;
    for (int it = 0; it < iters; it++) {
        const double* a = a0 + (it & (RING - 1)) * KC * LDSA;
        const double* b = b0 + (it & (RING - 1)) * KC * LDSB;
#pragma unroll
        for (int k0 = 0; k0 < KC; k0 += KS) {
            double rf[G][4], cf[G][4];
#pragma unroll
            for (int g = 0; g < G; g++)
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    rf[g][i] = a[(k0 + 4 * g) * LDSA + i * 8];
                    cf[g][i] = b[(k0 + 4 * g) * LDSB + i * 8];
                }
#pragma unroll
            for (int jj = 0; jj < 2; jj++)
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    double af[2 * G], bf[G];
#pragma unroll
                    for (int g = 0; g < G; g++) {
                        af[2 * g] = cf[g][2 * jj];
                        af[2 * g + 1] = cf[g][2 * jj + 1];
                        bf[g] = rf[g][i];
                    }
                    dmma16(acc[jj][i], af, bf);
                }
        }
    }
    double s = 0;
#pragma unroll
    for (int jj = 0; jj < 2; jj++)
#pragma unroll
        for (int i = 0; i < 4; i++) s += acc[jj][i][0] + acc[jj][i][1] + acc[jj][i][2] + acc[jj][i][3];
    if (s == 123.456) out[0] = s;
}

// flops_per_warp_iter: 2 * (warp tile rows) * (warp tile cols) * KC
template <typename Kern>
void run_kernel(Kern kern, const char* name, const char* shape, int rows, int cols, int warps, size_t smem,
                int ctas_per_sm, int sms, double* out, int iters) {
    // pad dynamic smem so that exactly ctas_per_sm CTAs fit
    size_t want = (ctas_per_sm == 1) ? 120 * 1024 : (ctas_per_sm == 2 ? 100 * 1024 : 60 * 1024);
    if (want > smem) smem = want;
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaFuncAttributes fa; CK(cudaFuncGetAttributes(&fa, kern));
    int fit = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, kern, warps * 32, smem));
    int blocks = sms * ctas_per_sm;
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    kern<<<blocks, warps * 32, smem>>>(out, iters); CK(cudaGetLastError()); CK(cudaDeviceSynchronize());
    float best = 1e30f;
    for (int r = 0; r < 3; r++) {
        CK(cudaEventRecord(e0)); kern<<<blocks, warps * 32, smem>>>(out, iters); CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1)); float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
    }
    double flops = (double)blocks * warps * iters * 2.0 * rows * cols * 16;
    printf("{\"variant\":\"%s\",\"shape\":\"%s\",\"warp_tile\":\"%dx%d\",\"warps\":%d,\"ctas_per_sm\":%d,"
           "\"ctas_per_sm_fit\":%d,\"regs\":%d,\"local_bytes\":%zu,\"tflops\":%.2f}\n",
           name, shape, rows, cols, warps, ctas_per_sm, fit, fa.numRegs, fa.localSizeBytes, flops / (best * 1e-3) / 1e12);
}

template <int RF, int CF, int WARPS, int LDSA, int LDSB>
void run(const char* name, int ctas_per_sm, int sms, double* out, int iters) {
    run_kernel(k_loop<RF, CF, WARPS, LDSA, LDSB>, name, "m8n8k4", RF * 8, CF * 8, WARPS, RING * 16 * (LDSA + LDSB) * 8,
               ctas_per_sm, sms, out, iters);
}

template <int KS, int MAXREG>
void run16(const char* name, const char* shape, int ctas_per_sm, int sms, double* out, int iters) {
    run_kernel(k_loop16<KS, MAXREG, 8, 132, 68>, name, shape, 32, 32, 8, RING * 16 * (132 + 68) * 8, ctas_per_sm, sms, out, iters);
}

int main(int argc, char** argv) {
    int iters = argc > 1 ? atoi(argv[1]) : 4000;
    cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
    int sms = p.multiProcessorCount;
    printf("device %s, %d SMs\n", p.name, sms);
    double* out; CK(cudaMalloc(&out, 8));
    run<4, 4, 8, 132, 68>("32x32 warp tile, 8 warps, 2 CTA/SM (gemm_nt.cu layout)", 2, sms, out, iters);
    run16<4, 112>("32x32 warp tile, 8 warps, 2 CTA/SM (gemm_nt.cu layout, 112 regs)", "m16n8k4", 2, sms, out, iters);
    run16<8, 112>("32x32 warp tile, 8 warps, 2 CTA/SM (gemm_nt.cu layout, 112 regs)", "m16n8k8", 2, sms, out, iters);
    run16<16, 112>("32x32 warp tile, 8 warps, 2 CTA/SM (gemm_nt.cu layout, 112 regs)", "m16n8k16", 2, sms, out, iters);
    run16<4, 255>("32x32 warp tile, 8 warps, 1 CTA/SM (no register cap)", "m16n8k4", 1, sms, out, iters);
    run16<8, 255>("32x32 warp tile, 8 warps, 1 CTA/SM (no register cap)", "m16n8k8", 1, sms, out, iters);
    run16<16, 255>("32x32 warp tile, 8 warps, 1 CTA/SM (no register cap)", "m16n8k16", 1, sms, out, iters);
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
