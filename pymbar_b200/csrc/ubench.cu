// On-box fp64 peaks used as the roofline denominators of the Hessian kernels (bench.py `roofline_hessian`).
// MEASURED_PEAKS.json (driver-written) holds HBM and bf16 figures only, so the fp64 ceiling is measured here, in
// the same process and under the same clocks as the kernel it bounds: a register-only loop of
// mma.sync.m8n8k4.f64 (SASS DMMA.8x8x4, 512 flop per warp instruction) and one of DFMA (64 flop per warp
// instruction), 16 warps per SM, 8 independent accumulator chains each.
#include "internal.cuh"

namespace mbar {

__global__ void __launch_bounds__(512) dmma_peak_kernel(double* out, int iters, double a, double b) {
    double c[8][2];
#pragma unroll
    for (int i = 0; i < 8; ++i) c[i][0] = c[i][1] = (double)i;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(c[i][0]), "+d"(c[i][1])
                         : "d"(a), "d"(b));
    }
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += c[i][0] + c[i][1];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void __launch_bounds__(512) dfma_peak_kernel(double* out, int iters, double a, double b) {
    double c[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) c[i] = (double)i + threadIdx.x * 1e-9;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) c[i] = fma(c[i], a, b);
    }
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += c[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

}  // namespace mbar

using namespace mbar;

extern "C" int mbar_b200_measure_fp64_peak(int device, double* dmma_tflops, double* dfma_tflops) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
        cudaGetLastError();
        set_error("no CUDA device %d", device);
        return MBAR_B200_ERR_NO_DEVICE;
    }
    MBAR_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    MBAR_CUDA(cudaGetDeviceProperties(&prop, device));
    const int sms = prop.multiProcessorCount;
    CallBuffers buf("measure_fp64_peak");
    double* d = nullptr;
    MBAR_TRY(buf.alloc(&d, (size_t)sms * 512));
    Events ev;
    MBAR_TRY(ev.create(2));
    const cudaEvent_t e0 = ev[0], e1 = ev[1];
    const int iters = 4096;
    double best[2] = {0.0, 0.0};
    for (int which = 0; which < 2; ++which) {
        for (int rep = 0; rep < 4; ++rep) {     // rep 0 warms up
            MBAR_CUDA(cudaEventRecord(e0));
            if (which == 0)
                dmma_peak_kernel<<<sms, 512>>>(d, iters, 1.0000001, 1e-9);
            else
                dfma_peak_kernel<<<sms, 512>>>(d, iters * 4, 1.0000001, 1e-9);
            MBAR_CUDA(cudaEventRecord(e1));
            MBAR_CUDA(cudaEventSynchronize(e1));
            float ms = 0.f;
            MBAR_CUDA(cudaEventElapsedTime(&ms, e0, e1));
            const double warpInst = (double)sms * 16.0 * 8.0 * (which == 0 ? iters : iters * 4);
            const double tf = warpInst * (which == 0 ? 512.0 : 64.0) / (ms * 1e-3) / 1e12;
            if (rep > 0 && tf > best[which]) best[which] = tf;
        }
    }
    MBAR_CUDA(cudaGetLastError());
    if (dmma_tflops) *dmma_tflops = best[0];
    if (dfma_tflops) *dfma_tflops = best[1];
    return MBAR_B200_OK;
}

extern "C" int mbar_b200_probe_exp(int device, int which, int64_t n, const double* a_host, double* out_host) {
    MBAR_REQUIRE(a_host && out_host && n >= 0, MBAR_B200_ERR_INVALID, "bad argument");
    MBAR_REQUIRE(which >= 0 && which <= 2, MBAR_B200_ERR_INVALID, "which=%d: 0, 1 or 2", which);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
        cudaGetLastError();
        set_error("no CUDA device %d", device);
        return MBAR_B200_ERR_NO_DEVICE;
    }
    if (n == 0) return MBAR_B200_OK;
    MBAR_CUDA(cudaSetDevice(device));
    CallBuffers buf("probe_exp");
    double* d = nullptr;
    MBAR_TRY(buf.alloc(&d, 2 * (size_t)n));
    int rc = MBAR_B200_OK;
    if (cudaMemcpy(d, a_host, (size_t)n * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess) {
        set_error("probe_exp: H2D copy failed");
        rc = MBAR_B200_ERR_CUDA;
    }
    if (rc == MBAR_B200_OK) rc = probe_exp_launch(which, n, d, d + n);
    if (rc == MBAR_B200_OK &&
        cudaMemcpy(out_host, d + n, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess) {
        set_error("probe_exp: D2H copy failed");
        rc = MBAR_B200_ERR_CUDA;
    }
    cudaGetLastError();
    return rc;
}
