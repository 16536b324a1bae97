// spec.cu — 30-band 1/3-octave spectrum bank (12th-order Butterworth band-passes in fp64).
//
// Replaces spectrum_instantiate / spectrum_run (src/spectrumlv2.c:73-121,159-257) over
// bandpass_setup / bandpass_process / proc_one (src/spectr.c:68-206) for N plugin instances.
// Design: one warp per instance, lane = band (30 of 32 lanes), the six transposed-DF-II
// biquad states and the band's coefficients live in fp64 registers, the (L+R)/2 input (plus the
// alternating +-1e-12 anti-denormal bias) is converted to double once per frame by the staging
// lanes and broadcast from shared memory.  The filter design itself runs on the host in complex
// double arithmetic in the reference's operation order (bitwise-equal coefficients).
// fp64 arithmetic keeps the reference's rounding sequence: products and sums are separate
// roundings except where a fused op is provably identical (multiplication by 1.0 and +-2.0).
#include <math.h>
#include <stdlib.h>
#include <complex>
#include <vector>
#include "common.cuh"

namespace b200m {

constexpr int SPEC_BANDS = 30;
constexpr int SPEC_TC = 64;               // frames per staged chunk
constexpr int SPEC_WARPS = 4;             // instances per CTA

struct SpecRun { int ac0; int nchan; };
// per-instance run parameters of one call, designed on the host from the instance's control ports (spec_control)
struct SpecCtl { float omega; int flags; };
constexpr int SPEC_CLEAR_MAX = 1, SPEC_REINIT_GUI = 2, SPEC_PARITY = 4;   // SPEC_PARITY: the instance's `ac` phase against the bank's frame count

// coef[band][16]: stage0 {b0,b1,b2,a1,a2}, stages 1..5 {a1,a2}; pad to 16
// FMA = B200M_PREC_FMA: the same transposed-DF-II cascade with fused multiply-adds (25 instead of 39 fp64 instructions per frame and
// band).  Band levels feed no integer result and the filters run in double precision, so the ports move by ~1e-12 dB, far inside the
// contract's +-1e-4 dB (tests/test_cor_spec_gpu.py::test_spec_fma_mode_within_tolerance).
template <bool FMA>
__global__ void __launch_bounds__ (SPEC_WARPS * 32)
spec_kernel (const float* __restrict__ in, size_t stride, int n_inst, int nfram, SpecRun rp, const SpecCtl* __restrict__ ctl, const double* __restrict__ coef,
             double* __restrict__ zst /* [inst][12][32] */, float* __restrict__ valf /* [inst][2][32] */, float* __restrict__ ports /* [inst][60] */)
{
    __shared__ float raw[SPEC_WARPS][2][2][SPEC_TC];      // [warp][stage][channel][frame]
    __shared__ double dd[SPEC_WARPS][SPEC_TC];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int inst = blockIdx.x * SPEC_WARPS + w;
    if (inst >= n_inst) return;                            // warp-uniform; no block-wide barriers below
    const int band = min (lane, SPEC_BANDS - 1);
    const bool live = lane < SPEC_BANDS;
    const float* pl = in + (size_t)inst * rp.nchan * stride;
    const float* pr = rp.nchan == 2 ? pl + stride : pl;
    const int nchunks = (nfram + SPEC_TC - 1) / SPEC_TC;

    auto issue = [&] (int c) {
        if (c < nchunks) {
            const int s0 = c * SPEC_TC;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = lane + 32 * h;
                const bool ok = (s0 + j) < nfram;
                cp_async4 (&raw[w][c & 1][0][j], ok ? pl + s0 + j : in, ok ? 4 : 0);
                cp_async4 (&raw[w][c & 1][1][j], ok ? pr + s0 + j : in, ok ? 4 : 0);
            }
        }
        cp_async_commit ();
    };
    issue (0);

    const double* cf = coef + band * 16;
    const double b0 = cf[0], b1 = cf[1], b2 = cf[2];
    double a1[6], a2[6], z1[6], z2[6];
    a1[0] = cf[3]; a2[0] = cf[4];
#pragma unroll
    for (int s = 1; s < 6; ++s) { a1[s] = cf[3 + 2 * s]; a2[s] = cf[4 + 2 * s]; }
    double* zp = zst + (size_t)inst * 12 * 32 + lane;
#pragma unroll
    for (int s = 0; s < 6; ++s) { z1[s] = zp[(2 * s) * 32]; z2[s] = zp[(2 * s + 1) * 32]; }
    float val = valf[(size_t)inst * 64 + lane], mx = valf[(size_t)inst * 64 + 32 + lane];
    const SpecCtl cp = ctl[inst];
    if (cp.flags & SPEC_CLEAR_MAX) mx = 0.0f;              // peak-hold reset (src/spectrumlv2.c:192-203)
    const float omega = cp.omega;
    const int ac0 = rp.ac0 ^ ((cp.flags & SPEC_PARITY) ? 1 : 0);

    for (int c = 0; c < nchunks; ++c) {
        const int s0 = c * SPEC_TC;
        const int len = min (SPEC_TC, nfram - s0);
        cp_async_wait<0> ();
        __syncwarp ();
        // staging: in = (L + R) / 2.0f ; out = in + (ac ? 1e-12 : -1e-12), ac toggling per frame from false
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int j = lane + 32 * h;
            const float l = raw[w][c & 1][0][j], r = raw[w][c & 1][1][j];
            const float x = rp.nchan == 2 ? __fmul_rn (__fadd_rn (l, r), 0.5f) : l;      // x/2.0f == x*0.5f exactly
            const bool ac = (((ac0 + s0 + j) & 1) == 0);
            dd[w][j] = __dadd_rn ((double)x, ac ? 1e-12 : -1e-12);
        }
        __syncwarp ();
        issue (c + 1);
#pragma unroll 2
        for (int j = 0; j < len; ++j) {
            double x = dd[w][j];
            if (FMA) {
                {
                    const double y = __fma_rn (b0, x, z1[0]);
                    z1[0] = __fma_rn (b1, x, __fma_rn (-a1[0], y, z2[0]));
                    z2[0] = __fma_rn (-a2[0], y, __dmul_rn (b2, x));
                    x = y;
                }
#pragma unroll
                for (int s = 1; s < 6; ++s) {
                    const double y = __dadd_rn (x, z1[s]);
                    z1[s] = __fma_rn ((s & 1) ? -2.0 : 2.0, x, __fma_rn (-a1[s], y, z2[s]));
                    z2[s] = __fma_rn (-a2[s], y, x);
                    x = y;
                }
            } else {
            // stage 0: general numerator (carries the pass-band normalisation, spectr.c:191-194)
            {
                const double y = __dadd_rn (__dmul_rn (b0, x), z1[0]);
                z1[0] = __dadd_rn (__dsub_rn (__dmul_rn (b1, x), __dmul_rn (a1[0], y)), z2[0]);
                z2[0] = __dsub_rn (__dmul_rn (b2, x), __dmul_rn (a2[0], y));
                x = y;
            }
            // stages 1..5: b = (1, +-2, 1): 1.0*x == x and fl(+-2x - t) == fma(+-2, x, -t) exactly
#pragma unroll
            for (int s = 1; s < 6; ++s) {
                const double y = __dadd_rn (x, z1[s]);
                const double t = __dmul_rn (a1[s], y);
                const double u = __fma_rn ((s & 1) ? -2.0 : 2.0, x, -t);
                z1[s] = __dadd_rn (u, z2[s]);
                z2[s] = __dsub_rn (x, __dmul_rn (a2[s], y));
                x = y;
            }
            }
            const float v = __double2float_rn (x);
            const float sq = __fmul_rn (v, v);
            val = __fadd_rn (val, __fmul_rn (omega, __fsub_rn (sq, val)));
            if (val > mx) mx = val;
        }
        __syncwarp ();
    }
    cp_async_wait<0> ();
    // end of run (:229-249): scrubs, anti-denormal bias, dB ports
    if (!finitef_ (val)) val = 0;
    if (!finitef_ (mx)) mx = 0;
#pragma unroll
    for (int s = 0; s < 6; ++s) {
        if (!(fabs (z1[s]) <= 1.7976931348623157e308)) z1[s] = 0;
        if (!(fabs (z2[s]) <= 1.7976931348623157e308)) z2[s] = 0;
    }
    if (live) {
#pragma unroll
        for (int s = 0; s < 6; ++s) { zp[(2 * s) * 32] = z1[s]; zp[(2 * s + 1) * 32] = z2[s]; }
        valf[(size_t)inst * 64 + lane] = __fadd_rn (val, 1e-20f);
        valf[(size_t)inst * 64 + 32 + lane] = mx;
        const float vs = __fsqrt_rn (__double2float_rn (__dmul_rn (2.0, (double)val)));
        const float ms = __fsqrt_rn (__double2float_rn (__dmul_rn (2.0, (double)mx)));
        ports[(size_t)inst * 60 + lane] = vs > .00001f ? __double2float_rn (__dmul_rn (20.0, (double)log10f_glibc (vs))) : -100.0f;
        // while a peak-reset handshake is pending the reference emits -500 - (rand() & 0xffff) to force a
        // GUI parameter change (:243-246); the engine emits the deterministic -500
        ports[(size_t)inst * 60 + 30 + lane] = (cp.flags & SPEC_REINIT_GUI) ? -500.0f
                                             : (ms > .00001f ? __double2float_rn (__dmul_rn (20.0, (double)log10f_glibc (ms))) : -100.0f);
    }
}

}  // namespace b200m

using namespace b200m;

struct b200m_spec {
    int device; uint32_t n_inst, nchan; double rate;
    uint64_t frames;                                      // frames processed by the bank: the `ac` phase of an instance never cleared
    std::vector<float> rst_h, spd_h;                      // per-instance control state (src/spectrumlv2.c:52-62)
    std::vector<SpecCtl> ctl;                             // host copy of d_ctl; [ctl_lo, ctl_hi) not uploaded yet
    SpecCtl* d_ctl = nullptr; uint32_t ctl_lo = 0, ctl_hi = 0;
    double W[30][6][6];                                   // a0 a1 a2 b0 b1 b2 per stage, as the reference stores them
    double *d_coef = nullptr, *d_z = nullptr; float *d_val = nullptr, *d_ports = nullptr;
    cudaStream_t own = nullptr; HostStage stage; bool last_host = false;
    int fma = 0;                                          // B200M_PREC_FMA
};

typedef std::complex<double> cplx;

// Band-pass design; restates bandpass_setup (src/spectr.c:89-206): Butterworth low-pass prototype poles ->
// band-pass via the (c_a, c_b) bilinear substitution -> per-section a1 = -2 Re(P), a2 = |P|^2, numerator
// (1, +-2, 1) -> unity gain at the geometric centre folded into section 0.  Same operation order and the
// same std::complex<double> operators as the reference, hence bitwise-equal coefficients on the same libm.
// noinline/noclone keeps `order` a run-time value: a clone specialised for order = 6 would let GCC fold the
// pole angles' cos/sin at compile time (MPFR, correctly rounded), which differs from glibc's run-time cos/sin
// in the last ulp for some angles — the reference build evaluates them at run time.
__attribute__ ((noinline, noclone))
static void design_band (double W[6][6], double rate, double freq, double band, int order)
{
    const double wc = 2. * M_PI * freq / rate, ww = 2. * M_PI * band / rate;
    double wl = wc - (ww / 2.), wu = wc + (ww / 2.);
    if (wu > M_PI - 1e-9) wu = M_PI - 1e-9;               // band limited to below nyquist (:113-122)
    if (wl < 1e-9) wl = 1e-9;                             // :123-132
    wu *= .5; wl *= .5;
    const double ca = cos (wu + wl) / cos (wu - wl);
    const double cb = 1. / tan (wu - wl);
    const double wn = 2. * atan (sqrt (tan (wu) * tan (wl)));
    const double ca2 = ca * ca, cb2 = cb * cb, ab2 = 2. * ca * cb;
    const cplx J (0.0, 1.0);
    for (int i = 0; i < order / 2; ++i) {
        const double th = M_PI_2 + (2 * i + 1) * M_PI / (2. * (double)order);
        cplx pole = cos (th) + J * sin (th);
        const cplx c = (1. + pole) / (1. - pole);
        const cplx d = 2 * (cb - 1) * c + 2 * (1 + cb);
        cplx v = (4 * (cb2 * (ca2 - 1) + 1)) * c;
        v += 8 * (cb2 * (ca2 - 1) - 1);
        v *= c;
        v += 4 * (cb2 * (ca2 - 1) + 1);
        v = std::sqrt (v);
        const cplx u0 = ab2 + std::real (v * -1.) + ab2 * std::real (c) + J * (std::imag (v * -1.) + ab2 * std::imag (c));
        const cplx u1 = ab2 + std::real (v) + ab2 * std::real (c) + J * (std::imag (v) + ab2 * std::imag (c));
        const cplx P[2] = {u0 / d, u1 / d};
        for (int k = 0; k < 2; ++k) {
            double* F = W[2 * i + k];
            F[0] = 1.;
            F[1] = -2 * std::real (P[k]);
            F[2] = std::real (P[k]) * std::real (P[k]) + std::imag (P[k]) * std::imag (P[k]);
            F[3] = 1.; F[4] = k ? -2. : 2.; F[5] = 1.;
        }
    }
    const double cw = cos (-wn), sw = sin (-wn), cw2 = cos (-2. * wn), sw2 = sin (-2. * wn);
    cplx num = 1, den = 1;
    for (int s = 0; s < order; ++s) {
        num *= ((1 + W[s][4] * cw) + cw2) + J * ((W[s][4] * sw) + sw2);
        den *= ((1 + W[s][1] * cw) + W[s][2] * cw2) + J * ((W[s][1] * sw) + W[s][2] * sw2);
    }
    const cplx scale = den / num;
    W[0][3] *= std::real (scale); W[0][4] *= std::real (scale); W[0][5] *= std::real (scale);
}

static void design_bank (double W[30][6][6], double rate)
{
    // band table (src/spectrumlv2.c:100-118): f_m = 1000 * 2^((i-16)/3), band edges at 2^(+-1/6), order 6
    const double f_r = 1000, b = 3;
    const double lo = pow (2, -1. / (2. * b)), hi = pow (2, 1. / (2. * b));
    for (int i = 0; i < SPEC_BANDS; ++i) {
        const int x = i - 16;
        const double f_m = pow (2, x / b) * f_r;
        const double f_1 = f_m * lo, f_2 = f_m * hi;
        design_band (W[i], rate, f_m, f_2 - f_1, 6);
    }
}

static float spec_omega (float speed, double rate)
{
    // 1.0 - e^(-2 pi v / rate), float result of a double argument (src/spectrumlv2.c:98,176)
    return 1.0f - expf (-2.0 * M_PI * speed / rate);
}

static cudaStream_t spec_stream (b200m_spec* h, void* stream) { return h->last_host ? h->own : (cudaStream_t)stream; }

// control-port handling at the top of spectrum_run (:170-205) for one instance: updates its state, returns its run parameters
static SpecCtl spec_control (b200m_spec* h, uint32_t i, float speed, float reset)
{
    SpecCtl c = {h->ctl[i].omega, h->ctl[i].flags & SPEC_PARITY};
    if (h->spd_h[i] != speed) {
        h->spd_h[i] = speed;
        float v = h->spd_h[i];
        if (v < 0.01) v = 0.01;
        if (v > 15.0) v = 15.0;
        c.omega = spec_omega (v, h->rate);
        h->rst_h[i] = 0;
    }
    if (h->rst_h[i] != reset) {
        if (fabsf (reset) < 3 || h->rst_h[i] == 0) c.flags |= SPEC_REINIT_GUI | SPEC_CLEAR_MAX;
        if (fabsf (reset) != 3) h->rst_h[i] = reset;
    }
    if (fabsf (reset) == 3) c.flags |= SPEC_REINIT_GUI;
    return c;
}

static void spec_mark (b200m_spec* h, uint32_t lo, uint32_t hi)
{
    if (h->ctl_lo >= h->ctl_hi) { h->ctl_lo = lo; h->ctl_hi = hi; }
    else { if (lo < h->ctl_lo) h->ctl_lo = lo; if (hi > h->ctl_hi) h->ctl_hi = hi; }
}

// an instance as b200m_spec_create leaves it (:95-98): rst_h = -4, spd_h = 1, `ac` from false at its next frame
static void spec_reset_ctl (b200m_spec* h, uint32_t i)
{
    h->rst_h[i] = -4; h->spd_h[i] = 1.0f;
    h->ctl[i].omega = spec_omega (1.0f, h->rate);
    h->ctl[i].flags = (h->frames & 1) ? SPEC_PARITY : 0;
}

// ctl[i * cstride] = {speed, reset} of instance i; cstride = 0: the same pair for every instance.  Only the instances whose run
// parameters changed are uploaded (one copy of the changed range, on the call's stream).
static int spec_process (b200m_spec* h, const float* d_in, size_t stride, uint32_t nfram, const float* ctl, size_t cstride, cudaStream_t st)
{
    for (uint32_t i = 0; i < h->n_inst; ++i) {
        const SpecCtl c = spec_control (h, i, ctl[i * cstride], ctl[i * cstride + 1]);
        if (memcmp (&c, &h->ctl[i], sizeof (c))) { h->ctl[i] = c; spec_mark (h, i, i + 1); }
    }
    if (h->ctl_lo < h->ctl_hi) {
        B200M_CUDA (cudaMemcpyAsync (h->d_ctl + h->ctl_lo, h->ctl.data () + h->ctl_lo, (h->ctl_hi - h->ctl_lo) * sizeof (SpecCtl), cudaMemcpyHostToDevice, st));
        h->ctl_lo = h->ctl_hi = 0;
    }
    SpecRun rp; rp.nchan = (int)h->nchan;
    rp.ac0 = (int)(h->frames & 1);
    h->frames += nfram;
    if (h->fma) spec_kernel<true><<<(h->n_inst + SPEC_WARPS - 1) / SPEC_WARPS, SPEC_WARPS * 32, 0, st>>> (
        d_in, stride, (int)h->n_inst, (int)nfram, rp, h->d_ctl, h->d_coef, h->d_z, h->d_val, h->d_ports);
    else spec_kernel<false><<<(h->n_inst + SPEC_WARPS - 1) / SPEC_WARPS, SPEC_WARPS * 32, 0, st>>> (
        d_in, stride, (int)h->n_inst, (int)nfram, rp, h->d_ctl, h->d_coef, h->d_z, h->d_val, h->d_ports);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

extern "C" {

int b200m_design_spec (double rate, double* W1080)
{
    if (!W1080 || !(rate >= 1000.0)) return set_err (B200M_E_INVAL, "bad argument");
    design_bank (reinterpret_cast<double (*)[6][6]> (W1080), rate);
    return 0;
}

int b200m_spec_create (b200m_spec** out, int device, uint32_t n_inst, uint32_t nchan, double rate)
{
    if (!out) return set_err (B200M_E_INVAL, "NULL out pointer");
    *out = nullptr;
    if (n_inst == 0 || !(rate >= 1000.0) || nchan < 1 || nchan > 2) return set_err (B200M_E_INVAL, "bad n_inst/nchan/rate");
    if (b200m_device_count () <= 0) return set_err (B200M_E_NODEVICE, "no CUDA device: b200meters has no CPU path");
    DeviceGuard g (device);
    if (!g.ok) return set_err (B200M_E_NODEVICE, "cannot select CUDA device %d", device);
    b200m_spec* h = new (std::nothrow) b200m_spec;
    if (!h) return set_err (B200M_E_NOMEM, "host allocation failed");
    h->device = device; h->n_inst = n_inst; h->nchan = nchan; h->rate = rate; h->frames = 0;
    h->rst_h.resize (n_inst); h->spd_h.resize (n_inst); h->ctl.resize (n_inst);
    for (uint32_t i = 0; i < n_inst; ++i) spec_reset_ctl (h, i);
    double coef[SPEC_BANDS][16];
    memset (coef, 0, sizeof (coef));
    design_bank (h->W, rate);
    for (int i = 0; i < SPEC_BANDS; ++i) {
        coef[i][0] = h->W[i][0][3]; coef[i][1] = h->W[i][0][4]; coef[i][2] = h->W[i][0][5];
        for (int s = 0; s < 6; ++s) { coef[i][3 + 2 * s] = h->W[i][s][1]; coef[i][4 + 2 * s] = h->W[i][s][2]; }
    }
    cudaError_t e = cudaSuccess;
    auto A = [&] (void** p, size_t bytes) { if (e == cudaSuccess) { e = cudaMalloc (p, bytes); if (e == cudaSuccess) e = cudaMemset (*p, 0, bytes); } };
    A ((void**)&h->d_coef, sizeof (coef));
    A ((void**)&h->d_z, (size_t)n_inst * 12 * 32 * sizeof (double));
    A ((void**)&h->d_val, (size_t)n_inst * 64 * sizeof (float));
    A ((void**)&h->d_ports, (size_t)n_inst * 60 * sizeof (float));
    A ((void**)&h->d_ctl, (size_t)n_inst * sizeof (SpecCtl));
    if (e == cudaSuccess) e = cudaMemcpy (h->d_coef, coef, sizeof (coef), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy (h->d_ctl, h->ctl.data (), (size_t)n_inst * sizeof (SpecCtl), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags (&h->own, cudaStreamNonBlocking);
    if (e != cudaSuccess) { int rc = cuda_fail (e, "spec_create", __FILE__, __LINE__); b200m_spec_destroy (h); return rc; }
    *out = h;
    return 0;
}

int b200m_spec_destroy (b200m_spec* h)
{
    if (!h) return 0;
    DeviceGuard g (h->device);
    cudaDeviceSynchronize ();
    cudaFree (h->d_coef); cudaFree (h->d_z); cudaFree (h->d_val); cudaFree (h->d_ports); cudaFree (h->d_ctl); h->stage.release ();
    if (h->own) cudaStreamDestroy (h->own);
    delete h;
    return 0;
}

int b200m_spec_process_ctl_device (b200m_spec* h, const float* d_in, size_t stride, uint32_t nfram, const float* ctl, void* stream)
{
    if (int rc = check_block_args (h, d_in, stride, nfram)) return rc;
    if (!ctl) return set_err (B200M_E_INVAL, "NULL ctl");
    DeviceGuard g (h->device);
    h->last_host = false;
    return spec_process (h, d_in, stride, nfram, ctl, 2, (cudaStream_t)stream);
}

int b200m_spec_process_device (b200m_spec* h, const float* d_in, size_t stride, uint32_t nfram, float speed, float reset, void* stream)
{
    if (int rc = check_block_args (h, d_in, stride, nfram)) return rc;
    DeviceGuard g (h->device);
    h->last_host = false;
    const float c[2] = {speed, reset};
    return spec_process (h, d_in, stride, nfram, c, 0, (cudaStream_t)stream);
}

static int spec_process_host (b200m_spec* h, const float* in, size_t stride, uint32_t nfram, const float* ctl, size_t cstride)
{
    if (int rc = check_block_args (h, in, stride, nfram)) return rc;
    DeviceGuard g (h->device);
    B200M_ENTER_HOST_PATH (h);
    const size_t nch = (size_t)h->n_inst * h->nchan;
    if (h->stage.ensure (nch, nfram)) return set_err (B200M_E_NOMEM, "staging buffer allocation failed");
    B200M_CUDA (cudaMemcpy2DAsync (h->stage.d, h->stage.cap * sizeof (float), in, stride * sizeof (float),
                                   (size_t)nfram * sizeof (float), nch, cudaMemcpyHostToDevice, h->own));
    h->last_host = true;
    return spec_process (h, h->stage.d, h->stage.cap, nfram, ctl, cstride, h->own);
}

int b200m_spec_process_ctl_host (b200m_spec* h, const float* in, size_t stride, uint32_t nfram, const float* ctl)
{
    if (!ctl) return set_err (B200M_E_INVAL, "NULL ctl");
    return spec_process_host (h, in, stride, nfram, ctl, 2);
}

int b200m_spec_process_host (b200m_spec* h, const float* in, size_t stride, uint32_t nfram, float speed, float reset)
{
    const float c[2] = {speed, reset};
    return spec_process_host (h, in, stride, nfram, c, 0);
}

int b200m_spec_clear (b200m_spec* h, int32_t inst, void* stream)
{
    if (!h || inst < -1 || inst >= (int32_t)h->n_inst) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    cudaStream_t st = spec_stream (h, stream);
    const uint32_t i0 = inst < 0 ? 0 : (uint32_t)inst, n = inst < 0 ? h->n_inst : 1;
    // filter states, val / max and the ports as b200m_spec_create zeroes them
    B200M_CUDA (cudaMemsetAsync (h->d_z + (size_t)i0 * 12 * 32, 0, (size_t)n * 12 * 32 * sizeof (double), st));
    B200M_CUDA (cudaMemsetAsync (h->d_val + (size_t)i0 * 64, 0, (size_t)n * 64 * sizeof (float), st));
    B200M_CUDA (cudaMemsetAsync (h->d_ports + (size_t)i0 * 60, 0, (size_t)n * 60 * sizeof (float), st));
    for (uint32_t i = i0; i < i0 + n; ++i) spec_reset_ctl (h, i);
    spec_mark (h, i0, i0 + n);                             // uploaded by the next process call, on its stream
    return 0;
}

int b200m_spec_set_precision (b200m_spec* h, int mode)
{
    if (!h || (mode != B200M_PREC_EXACT && mode != B200M_PREC_FMA)) return set_err (B200M_E_INVAL, "bad argument");
    h->fma = mode == B200M_PREC_FMA;                       // takes effect with the next process call
    return 0;
}

int b200m_spec_results (b200m_spec* h, float* out60, void* stream)
{
    if (!h || !out60) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = spec_stream (h, stream);
    B200M_CUDA (cudaMemcpyAsync (out60, h->d_ports, (size_t)h->n_inst * 60 * sizeof (float), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_spec_state (b200m_spec* h, uint32_t inst, double* z360, float* val30, float* max30, void* stream)
{
    if (!h || !z360 || !val30 || !max30 || inst >= h->n_inst) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    cudaStream_t st = spec_stream (h, stream);
    double zt[12 * 32]; float vt[64];
    B200M_CUDA (cudaMemcpyAsync (zt, h->d_z + (size_t)inst * 12 * 32, sizeof (zt), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaMemcpyAsync (vt, h->d_val + (size_t)inst * 64, sizeof (vt), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    for (int b = 0; b < 30; ++b) {
        for (int s = 0; s < 6; ++s) { z360[(b * 6 + s) * 2] = zt[(2 * s) * 32 + b]; z360[(b * 6 + s) * 2 + 1] = zt[(2 * s + 1) * 32 + b]; }
        val30[b] = vt[b]; max30[b] = vt[32 + b];
    }
    return 0;
}

int b200m_spec_coeffs (const b200m_spec* h, double* W1080)
{
    if (!h || !W1080) return set_err (B200M_E_INVAL, "NULL argument");
    memcpy (W1080, h->W, sizeof (h->W));
    return 0;
}

}  // extern "C"
