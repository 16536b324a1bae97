// selftest.cu — device-side evaluation hooks for the parity tests (no DSP state, no bank).
//
// b200m_selftest_log10f evaluates the engine's glibc-exact log10f (common.cuh: log10f_glibc, the function every loudness
// value, dB port and histogram bin of the engine goes through; reference call sites ebumeter/ebu_r128_proc.cc:116-141,259)
// on a contiguous range of float BIT PATTERNS, so that a test can sweep all 2^31 non-negative floats against the host
// libm's log10f (tests/test_log10f_sweep_gpu.py).
#include "common.cuh"

namespace b200m {

__global__ void selftest_log10f_kernel (uint32_t first, uint32_t count, float* __restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) out[i] = log10f_glibc (__uint_as_float (first + (uint32_t)i));
}

}  // namespace b200m

using namespace b200m;

extern "C" int b200m_selftest_log10f (int device, uint32_t first_bits, uint32_t count, float* d_out, void* stream)
{
    if (!d_out || count == 0) return set_err (B200M_E_INVAL, "bad argument");
    if (b200m_device_count () <= 0) return set_err (B200M_E_NODEVICE, "no CUDA device");
    DeviceGuard g (device);
    if (!g.ok) return set_err (B200M_E_NODEVICE, "cannot select CUDA device %d", device);
    selftest_log10f_kernel<<<(count + 255) / 256, 256, 0, (cudaStream_t)stream>>> (first_bits, count, d_out);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}
