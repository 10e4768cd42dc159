// Standalone driver for the product's DMMA NT kernel (unity-includes gemm_nt.cu): sweeps K and
// beta to separate main-loop efficiency from per-tile prologue/epilogue costs.
#include "../stheno.jl_b200/csrc/gemm_nt.cu"
#include <cstdio>
#include <vector>
namespace sb { thread_local int64_t g_launch_count = 0; void set_error(const std::string&) {} int32_t cuda_fail(cudaError_t, const char*, const char*, int) { return -2; } }
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)
int main(int argc, char** argv) {
    long long onlyK = argc > 1 ? atoll(argv[1]) : 0; double onlyBeta = argc > 2 ? atof(argv[2]) : -1;
    const int64_t M = 16384, N = 16384;
    const int64_t KMAX = 4096;
    double *A, *B, *C;
    CK(cudaMalloc(&A, M * KMAX * 8)); CK(cudaMalloc(&B, N * KMAX * 8)); CK(cudaMalloc(&C, M * N * 8));
    CK(cudaMemset(A, 0, M * KMAX * 8)); CK(cudaMemset(B, 0, N * KMAX * 8)); CK(cudaMemset(C, 0, M * N * 8));
    {   // the kernel is built around 2 CTAs per SM (one CTA's epilogue overlaps the other's main loop)
        CK(cudaFuncSetAttribute(sb::gemm_nt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sb::SMEM_BYTES));
        cudaFuncAttributes fa; CK(cudaFuncGetAttributes(&fa, sb::gemm_nt_kernel));
        int fit = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, sb::gemm_nt_kernel, sb::THREADS, sb::SMEM_BYTES));
        printf("{\"kernel\":\"gemm_nt_kernel\",\"regs\":%d,\"local_bytes\":%zu,\"smem_bytes\":%zu,\"ctas_per_sm\":%d}\n",
               fa.numRegs, fa.localSizeBytes, sb::SMEM_BYTES, fit);
    }
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    for (double beta : {1.0, 0.0})
        for (int64_t K : {128, 256, 512, 1024, 4096}) {
            if (onlyK && (K != onlyK || beta != onlyBeta)) continue;
            sb::launch_gemm_nt(A, M, B, N, C, M, M, N, K, -1.0, beta, 0); CK(cudaDeviceSynchronize());
            CK(cudaEventRecord(e0));
            int reps = K >= 1024 ? 1 : 3;
            for (int r = 0; r < reps; r++) sb::launch_gemm_nt(A, M, B, N, C, M, M, N, K, -1.0, beta, 0);
            CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
            float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); ms /= reps;
            printf("{\"M\":%lld,\"N\":%lld,\"K\":%lld,\"beta\":%.0f,\"ms\":%.3f,\"tflops\":%.2f}\n", (long long)M, (long long)N,
                   (long long)K, beta, ms, 2.0 * M * N * K / (ms * 1e-3) / 1e12);
        }
    return 0;
}
