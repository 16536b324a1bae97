// common.cuh — shared host/device helpers of the b200meters CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <new>

#include "../../include/b200meters.h"

namespace b200m {

// ---------------------------------------------------------------- host-side plumbing
extern thread_local char g_err[512];
extern std::atomic<uint64_t> g_launches;

int  set_err (int code, const char* fmt, ...);
int  cuda_fail (cudaError_t e, const char* what, const char* file, int line);

#define B200M_CUDA(call)                                                             \
    do {                                                                             \
        cudaError_t e_ = (call);                                                     \
        if (e_ != cudaSuccess) return b200m::cuda_fail (e_, #call, __FILE__, __LINE__); \
    } while (0)

#define B200M_LAUNCHED(n) (b200m::g_launches.fetch_add ((n), std::memory_order_relaxed))

// every bank pins its device on entry and restores the caller's device on exit
struct DeviceGuard {
    int prev = -1; bool ok = true;
    explicit DeviceGuard (int dev) {
        if (cudaGetDevice (&prev) != cudaSuccess) { ok = false; return; }
        if (prev != dev && cudaSetDevice (dev) != cudaSuccess) ok = false;
    }
    ~DeviceGuard () { if (prev >= 0) cudaSetDevice (prev); }
};

// device staging area for *_process_host: [channels][cap] floats, grown on demand
struct HostStage {
    float* d = nullptr; size_t chans = 0, cap = 0;
    int ensure (size_t channels, size_t n) {
        if (d && channels == chans && n <= cap) return 0;
        if (d) { cudaFree (d); d = nullptr; }
        size_t c = (n + 63) & ~size_t (63);
        if (cudaMalloc (&d, channels * c * sizeof (float)) != cudaSuccess) { d = nullptr; return B200M_E_NOMEM; }
        chans = channels; cap = c; return 0;
    }
    void release () { if (d) cudaFree (d); d = nullptr; }
};

int check_block_args (const void* h, const void* in, size_t stride, uint32_t nfram);

// A bank switches to its own stream with the first *_host call; whatever the caller queued before that (controls on the
// streams it passed) must not race with it: one device-wide synchronisation at the transition, nothing afterwards.
#define B200M_ENTER_HOST_PATH(h) do { if (!(h)->last_host) B200M_CUDA (cudaDeviceSynchronize ()); } while (0)

#ifdef __CUDACC__
// ---------------------------------------------------------------- device helpers
#define B200M_DEV __device__ __forceinline__

B200M_DEV bool finitef_ (float v) { return fabsf (v) <= 3.402823466e+38f; }   // false for NaN, +-Inf
B200M_DEV float scrub (float v) { return finitef_ (v) ? v : 0.0f; }           // "!isfinite(z) ? 0 : z"

// cp.async (LDGSTS): global -> shared without a register round trip
B200M_DEV void cp_async16 (void* smem, const void* gmem, int src_bytes) {
    unsigned s = (unsigned)__cvta_generic_to_shared (smem);
    asm volatile ("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(src_bytes));
}
B200M_DEV void cp_async4 (void* smem, const void* gmem, int src_bytes) {
    unsigned s = (unsigned)__cvta_generic_to_shared (smem);
    asm volatile ("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(s), "l"(gmem), "r"(src_bytes));
}
B200M_DEV void cp_async_commit () { asm volatile ("cp.async.commit_group;\n" ::); }
template <int N> B200M_DEV void cp_async_wait () { asm volatile ("cp.async.wait_group %0;\n" ::"n"(N)); }

// ---- log10f, bit-identical to glibc 2.39 libm ------------------------------------------
// The reference turns fragment powers into loudness with log10f (ebumeter/ebu_r128_proc.cc:259,
// :116-122,:140-141) and bins the result into INTEGER histograms (:66-79), so the engine needs
// the host libm's log10f to the last bit, not CUDA's 2-ulp one.  glibc 2.39's log10f is the
// fdlibm wrapper  z = y*log10_2lo + ivln10*logf(x'); return z + y*log10_2hi  (float arithmetic)
// around the table-driven double-precision logf of ARM's optimized-routines (16-entry table,
// degree-3 polynomial).  Both are restated here from the published algorithms; the table is the
// one in libm's __logf_data.  Checked exhaustively on the host (all 2^31 non-negative floats)
// against libm's logf and log10f in FMA and non-FMA form: 0 mismatches — see DESIGN.md §log10f
// and tests/test_libm_parity.py.
static __device__ __constant__ double c_logf_tab[16][2] = {
    {0x1.661ec79f8f3bep+0, -0x1.57bf7808caadep-2}, {0x1.571ed4aaf883dp+0, -0x1.2bef0a7c06ddbp-2},
    {0x1.49539f0f010bp+0, -0x1.01eae7f513a67p-2},  {0x1.3c995b0b80385p+0, -0x1.b31d8a68224e9p-3},
    {0x1.30d190c8864a5p+0, -0x1.6574f0ac07758p-3}, {0x1.25e227b0b8eap+0, -0x1.1aa2bc79c81p-3},
    {0x1.1bb4a4a1a343fp+0, -0x1.a4e76ce8c0e5ep-4}, {0x1.12358f08ae5bap+0, -0x1.1973c5a611cccp-4},
    {0x1.0953f419900a7p+0, -0x1.252f438e10c1ep-5}, {0x1p+0, 0x0p+0},
    {0x1.e608cfd9a47acp-1, 0x1.aa5aa5df25984p-5},  {0x1.ca4b31f026aap-1, 0x1.c5e53aa362eb4p-4},
    {0x1.b2036576afce6p-1, 0x1.526e57720db08p-3},  {0x1.9c2d163a1aa2dp-1, 0x1.bc2860d22477p-3},
    {0x1.886e6037841edp-1, 0x1.1058bc8a07ee1p-2},  {0x1.767dcf5534862p-1, 0x1.4043057b6ee09p-2}};

// logf for x with a normal, positive, finite bit pattern (the wrapper below guarantees it)
B200M_DEV float logf_glibc_normal (float x)
{
    uint32_t ix = __float_as_uint (x);
    if (ix == 0x3f800000u) return 0.0f;
    uint32_t tmp = ix - 0x3f330000u;
    int i = (tmp >> 19) & 15;
    int k = (int32_t)tmp >> 23;
    uint32_t iz = ix - (tmp & 0xff800000u);
    double invc = c_logf_tab[i][0], logc = c_logf_tab[i][1];
    double z = (double)__uint_as_float (iz);
    double r  = __fma_rn (z, invc, -1.0);
    double y0 = __fma_rn ((double)k, 0x1.62e42fefa39efp-1, logc);
    double r2 = __dmul_rn (r, r);
    double y  = __fma_rn (0x1.5575b0be00b6ap-2, r, -0x1.ffffef20a4123p-2);
    y = __fma_rn (-0x1.00ea348b88334p-2, r2, y);
    y = __fma_rn (y, r2, __dadd_rn (y0, r));
    return __double2float_rn (y);
}

B200M_DEV float log10f_glibc (float x)
{
    const float two25 = 3.3554432000e+07f, ivln10 = 4.3429449201e-01f;
    const float log10_2hi = 3.0102920532e-01f, log10_2lo = 7.9034151668e-07f;
    int32_t hx = __float_as_int (x), k = 0;
    if (hx < 0x00800000) {                                  // x < 2^-126, zero or negative
        if ((hx & 0x7fffffff) == 0) return __fdiv_rn (-two25, fabsf (x));      // -inf
        if (hx < 0) return __fdiv_rn (__fsub_rn (x, x), __fsub_rn (x, x));     // NaN
        k -= 25; x = __fmul_rn (x, two25); hx = __float_as_int (x);
    }
    if (hx >= 0x7f800000) return __fadd_rn (x, x);
    k += (hx >> 23) - 127;
    int32_t i = (int32_t)(((uint32_t)k & 0x80000000u) >> 31);
    hx = (hx & 0x007fffff) | ((0x7f - i) << 23);
    float y = (float)(k + i);
    float z = __fadd_rn (__fmul_rn (y, log10_2lo), __fmul_rn (ivln10, logf_glibc_normal (__int_as_float (hx))));
    return __fadd_rn (z, __fmul_rn (y, log10_2hi));
}
#endif  // __CUDACC__

}  // namespace b200m
