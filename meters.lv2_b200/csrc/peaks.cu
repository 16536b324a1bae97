// peaks.cu — on-device probes of the two ALU ceilings that bound the compute-bound metering kernels.
//
// The true-peak FIR is bound by fp32 *instruction issue* (unfused FMUL + FADD, the reference's rounding sequence forbids FMA) and the
// 1/3-octave bank by the fp64 pipe (SURVEY.md §8d).  bench.py reports each such kernel against these probes as
// well as against the HBM roofline.  Each probe runs independent dependent-chains of unfused multiply + add.
#include "common.cuh"

namespace b200m {

template <typename T>
__global__ void __launch_bounds__ (256) peak_probe_kernel (T* out, int iters, T k1, T k2)
{
    T a[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = (T)(threadIdx.x + i) * (T)1e-3;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                if (sizeof (T) == 4) a[i] = (T)__fadd_rn (__fmul_rn ((float)a[i], (float)k1), (float)k2);
                else a[i] = (T)__dadd_rn (__dmul_rn ((double)a[i], (double)k1), (double)k2);
            }
        }
    }
    T s = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += a[i];
    if (s == (T)123.456) out[0] = s;            // never true: keeps the chains alive
}

}  // namespace b200m

using namespace b200m;

extern "C" int b200m_peak_probe (int device, int kind, double* gops)
{
    if (!gops || kind < 0 || kind > 1) return set_err (B200M_E_INVAL, "bad argument");
    if (b200m_device_count () <= 0) return set_err (B200M_E_NODEVICE, "no CUDA device");
    DeviceGuard g (device);
    cudaDeviceProp pr; B200M_CUDA (cudaGetDeviceProperties (&pr, device));
    void* d; B200M_CUDA (cudaMalloc (&d, 64));
    const int iters = kind == 1 ? 1024 : 4096, blocks = pr.multiProcessorCount * 8;
    cudaEvent_t e0, e1; cudaEventCreate (&e0); cudaEventCreate (&e1);
    float best = 1e30f;
    for (int rep = 0; rep < 4; ++rep) {
        cudaEventRecord (e0);
        if (kind == 0) peak_probe_kernel<float><<<blocks, 256>>> ((float*)d, iters, 0.999f, 1e-3f);
        else peak_probe_kernel<double><<<blocks, 256>>> ((double*)d, iters, 0.999, 1e-3);
        B200M_LAUNCHED (1);
        cudaEventRecord (e1); cudaEventSynchronize (e1);
        float ms; cudaEventElapsedTime (&ms, e0, e1);
        if (rep && ms < best) best = ms;
    }
    cudaEventDestroy (e0); cudaEventDestroy (e1); cudaFree (d);
    B200M_CUDA (cudaGetLastError ());
    // lane-operations (one FMUL or FADD of one lane) per second, in units of 1e9
    *gops = (double)blocks * 256.0 * iters * 4 * 8 * 2 / (best * 1e-3) / 1e9;
    return 0;
}
