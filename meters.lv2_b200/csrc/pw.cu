// pw.cu — phasewheel / stereoscope FFT analysis bank (cuFFT-free mixed-radix Stockham kernel).
//
// Replaces, for N stereo instances, the GUI-side analysis of the phasewheel: fftx_init / fftx_run /
// ft_analyze (gui/fft.c:208-361, Hann window :69-79,122-161) for the left and right channel plus
// process_audio (gui/phasewheel.c:1307-1342; stereoscope: gui/stereoscope.c:705-741).  The reference calls FFTW3
// (fftwf_plan_r2r_1d R2HC, gui/fft.c:234) which is neither vendored nor pinned; this kernel computes the same DFT
// (X_k = sum x_n e^{-2 pi i nk/N}) in fp32 with its own algorithm, so parity for this bank is
// tolerance-based and pinned against an independent float64 FFT (numpy) in tests/test_pw_gpu.py.
// Every size the reference GUI offers is provided: fft_bins 64 .. 8192 and 6144 (N = 128 .. 16384 and 12288 = 3 * 4096,
// gui/phasewheel.c:1108-1116).
//
// Design: the ring buffers of all instances advance in lock step, so the host tracks the write
// offset and the 25 Hz analysis clock; one CTA per instance runs, per channel, an N/2-point complex autosort
// (Stockham) FFT in shared memory (radix-3 pass when 3 | N, radix-4 passes, one radix-2 pass when needed), splits it
// into the real spectrum, and writes phase difference / level bins with coalesced stores.  The block append can be
// fused with the stereo-correlation bank (b200m_pw_attach_cor): the input is then read from HBM once for both meters.
#include <math.h>
#include <stdlib.h>
#include "common.cuh"

namespace b200m {

constexpr int PW_THREADS = 256;

__global__ void pw_append_kernel (const float* __restrict__ in, size_t stride, int rows, int nfram, int N, int rboff,
                                  float* __restrict__ ring)
{
    // r_buf[(i + n_off) % n_siz] = data[i]  (gui/fft.c:302-305)
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)rows * nfram) return;
    const int row = (int)(idx / nfram), j = (int)(idx % nfram);
    int o = rboff + j; if (o >= N) o -= N;                                    // nfram <= N, rboff < N
    ring[(size_t)row * N + o] = in[(size_t)row * stride + j];
}

B200M_DEV float2 cmul (float2 a, float2 b) { return make_float2 (fmaf (a.x, b.x, -a.y * b.y), fmaf (a.x, b.y, a.y * b.x)); }
B200M_DEV float2 cadd (float2 a, float2 b) { return make_float2 (a.x + b.x, a.y + b.y); }
B200M_DEV float2 csub (float2 a, float2 b) { return make_float2 (a.x - b.x, a.y - b.y); }

// One autosort (Stockham) pass of radix R over M complex points: n = current sub-transform length, s = M / n its stride.
// tw[] holds the N = 2M-th roots of unity exp(-2 pi i k / N), so exp(-2 pi i p m / n) = tw[2 p m s].
// The stride is always s = s3 * 2^sh with s3 in {1, 3} (the radix-3 pass, if any, runs first), so t = p s + q splits with a
// shift, a mask and at most a division by the constant 3 instead of a run-time integer division.
template <int R>
B200M_DEV void stockham_pass (const float2* __restrict__ X, float2* __restrict__ Y, const float2* __restrict__ tw, int M, int n, int s3, int sh, int tid)
{
    const int n1 = n / R;
    const int s = s3 << sh;
    for (int t = tid; t < M / R; t += PW_THREADS) {
        int p, q;
        if (s3 == 1) { p = t >> sh; q = t & ((1 << sh) - 1); }
        else { const int u = t >> sh; p = u / 3; q = ((u - 3 * p) << sh) | (t & ((1 << sh) - 1)); }
        float2 a[R];
#pragma unroll
        for (int j = 0; j < R; ++j) a[j] = X[q + s * (p + j * n1)];
        float2 y[R];
        if (R == 2) { y[0] = cadd (a[0], a[1]); y[1] = csub (a[0], a[1]); }
        else if (R == 3) {
            const float2 t1 = cadd (a[1], a[2]);
            const float2 t2 = make_float2 (fmaf (-0.5f, t1.x, a[0].x), fmaf (-0.5f, t1.y, a[0].y));
            const float2 d = csub (a[1], a[2]);
            const float2 t3 = make_float2 (0.86602540378443865f * d.y, -0.86602540378443865f * d.x);   // -i sin(pi/3) (a1 - a2)
            y[0] = cadd (a[0], t1); y[1] = cadd (t2, t3); y[2] = csub (t2, t3);
        } else {
            const float2 apc = cadd (a[0], a[2]), amc = csub (a[0], a[2]), bpd = cadd (a[1], a[3]);
            const float2 jbmd = make_float2 (-(a[1].y - a[3].y), a[1].x - a[3].x);                     // i (b - d)
            y[0] = cadd (apc, bpd); y[1] = csub (amc, jbmd); y[2] = csub (apc, bpd); y[3] = cadd (amc, jbmd);
        }
        if (p != 0) {
#pragma unroll
            for (int m = 1; m < R; ++m) y[m] = cmul (tw[2 * p * m * s], y[m]);
        }
        if (R == 4 && s == 1) {
            // first pass of a power-of-two transform: the four outputs are contiguous -> two 16-byte stores instead of four 8-byte
            // stores at a 32-byte lane stride (4-way bank conflicts)
            float4* d = reinterpret_cast<float4*> (Y + 4 * p);
            d[0] = make_float4 (y[0].x, y[0].y, y[1].x, y[1].y);
            d[1] = make_float4 (y[2].x, y[2].y, y[3].x, y[3].y);
        } else {
#pragma unroll
            for (int m = 0; m < R; ++m) Y[q + s * (R * p + m)] = y[m];
        }
    }
}

// ring: [inst][2][N]; the oldest sample sits at offset `start`.  window: N floats.  tw[k] = exp(-2 pi i k / N), k < N.
// One CTA per instance.  Each channel's N-point real transform is computed as an M = N/2-point complex transform of
// z[n] = x[2n] + i x[2n+1] followed by the usual split  X[k] = E[k] + W_N^k O[k]  (E, O: transforms of the even / odd samples):
// half the shared memory of packing L + iR into one N-point transform, which is what lets N = 16384 (gui/phasewheel.c:1116)
// fit: 2 x M complex ping-pong buffers + the left channel's power / phase = 12 N bytes.
__global__ void __launch_bounds__ (PW_THREADS)
pw_analyze_kernel (const float* __restrict__ ring, int N, int f3, int f4, int f2, int start, const float* __restrict__ window,
                   const float2* __restrict__ tw, float db_thresh, float* __restrict__ rawp /* [inst][4][bins] or NULL */,
                   float* __restrict__ phase, float* __restrict__ level, float* __restrict__ peak, int mode)
{
    extern __shared__ __align__ (16) float2 sm[];          // X, Y: M complex each; then powL[bins], phL[bins]
    __shared__ float red[PW_THREADS / 32];
    const int M = N / 2, bins = N / 2;
    float2* bufA = sm; float2* bufB = sm + M;
    float* sPL = reinterpret_cast<float*> (sm + 2 * M); float* sFL = sPL + bins;
    const int inst = blockIdx.x, tid = threadIdx.x;
    float pk = 0.0f;
    for (int ch = 0; ch < 2; ++ch) {
        const float* rg = ring + ((size_t)inst * 2 + ch) * N;
        float2* X = bufA; float2* Y = bufB;
        // last N samples in time order, times the window (gui/fft.c:318-333), packed even / odd
        for (int t = tid; t < M; t += PW_THREADS) {
            int s0 = start + 2 * t; if (s0 >= N) s0 -= N;
            int s1 = s0 + 1; if (s1 >= N) s1 -= N;
            X[t] = make_float2 (__fmul_rn (rg[s0], window[2 * t]), __fmul_rn (rg[s1], window[2 * t + 1]));
        }
        __syncthreads ();
        int n = M, s3 = 1, sh = 0;                             // stride s = s3 << sh
        for (int i = 0; i < f3; ++i) { stockham_pass<3> (X, Y, tw, M, n, s3, sh, tid); __syncthreads (); float2* T = X; X = Y; Y = T; n /= 3; s3 *= 3; }
        for (int i = 0; i < f4; ++i) { stockham_pass<4> (X, Y, tw, M, n, s3, sh, tid); __syncthreads (); float2* T = X; X = Y; Y = T; n /= 4; sh += 2; }
        for (int i = 0; i < f2; ++i) { stockham_pass<2> (X, Y, tw, M, n, s3, sh, tid); __syncthreads (); float2* T = X; X = Y; Y = T; n /= 2; sh += 1; }
        // ft_analyze (gui/fft.c:163-180) for this channel, then (right channel) process_audio (gui/phasewheel.c:1313-1331)
        float* rp = rawp ? rawp + (size_t)inst * 4 * bins : nullptr;
        for (int k = tid; k < bins; k += PW_THREADS) {
            float pw_, ph_;
            if (k == 0) { const float x0 = X[0].x + X[0].y; pw_ = x0 * x0; ph_ = 0.0f; }          // power[0] = out[0]^2, phase[0] = 0
            else if (k == bins - 1) { pw_ = 0.0f; ph_ = 0.0f; }                                   // never written by ft_analyze (i < data_size - 1): stays as fftx_reset left it
            else {
                const float2 A = X[k], Bm = X[M - k], w = tw[k];
                const float er = 0.5f * (A.x + Bm.x), ei = 0.5f * (A.y - Bm.y);
                const float orr = 0.5f * (A.y + Bm.y), oi = -0.5f * (A.x - Bm.x);
                const float re = er + fmaf (w.x, orr, -w.y * oi), im = ei + fmaf (w.x, oi, w.y * orr);
                pw_ = fmaf (re, re, im * im);
                ph_ = (mode == 0 || rp) ? atan2f (im, re) : 0.0f;            // the stereoscope's process_audio never reads ft->phase
            }
            if (rp) { rp[ch * bins + k] = pw_; rp[(2 + ch) * bins + k] = ph_; }
            if (ch == 0) { sPL[k] = pw_; sFL[k] = ph_; continue; }
            const float pl = sPL[k], fl = sFL[k], pr = pw_, fr = ph_;
            if (k < 1 || k >= bins - 1) continue;
            if (mode == 1) {
                // stereoscope process_audio (gui/stereoscope.c:713-739): phase[] holds ui->lr[], both outputs are smoothed state
                float* lrp = phase + (size_t)inst * bins + k; float* lvp = level + (size_t)inst * bins + k;
                if (pl < 1e-20f && pr < 1e-20f) { *lrp = 0.5f; *lvp = 0.0f; }
                else {
                    const float lv = pl > pr ? pl : pr;
                    const float dq = __fsub_rn (__fsqrt_rn (pr), __fsqrt_rn (pl));
                    const float lr = __double2float_rn (.5 + __ddiv_rn (__dmul_rn (.5, (double)dq), (double)__fsqrt_rn (lv)));
                    const float l0 = *lvp, r0 = *lrp;
                    *lvp = __double2float_rn ((double)l0 + (__dmul_rn (.1, (double)__fsub_rn (lv, l0)) + 1e-20));
                    *lrp = __double2float_rn ((double)r0 + (__dmul_rn (.1, (double)__fsub_rn (lr, r0)) + 1e-10));
                }
            } else {
                float ph, lv;
                if (pl < db_thresh || pr < db_thresh) { ph = 0.0f; lv = -100.0f; }
                else { ph = __fsub_rn (fr, fl); lv = pl > pr ? pl : pr; if (lv > pk) pk = lv; }   // MAX(a,b) = a > b ? a : b
                phase[(size_t)inst * bins + k] = ph;
                level[(size_t)inst * bins + k] = lv;
            }
        }
        __syncthreads ();                                    // the buffers are reused by the right channel
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) pk = fmaxf (pk, __shfl_xor_sync (0xffffffffu, pk, o));
    if ((tid & 31) == 0) red[tid >> 5] = pk;
    __syncthreads ();
    if (tid == 0 && mode == 0) {
        for (int i = 1; i < PW_THREADS / 32; ++i) pk = fmaxf (pk, red[i]);
        // ui->peak += .04 * (peak - ui->peak) + 1e-15;  (double arithmetic on a float lvalue, :1333-1335)
        float up = peak[inst];
        up = __double2float_rn ((double)up + (.04 * (double)__fsub_rn (pk, up) + 1e-15));
        if (isnan (up)) up = 0;
        if (up > 1000) up = 1000;
        peak[inst] = up;
    }
}

__global__ void pw_init_kernel (size_t n, float* level, float* phase, float ph0) { const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; if (i < n) { level[i] = -100.0f; phase[i] = ph0; } }

}  // namespace b200m

using namespace b200m;

struct b200m_cor;
namespace b200m {
// cor.cu: one Stcorrdsp::process block for every pair of the bank; when `ring` is given the block is also appended to the
// phasewheel ring [pair][2][N] at offset rboff (fused feed: the input is read once)
int cor_feed (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, cudaStream_t st, float* ring, int N, int rboff);
uint32_t cor_instances (const b200m_cor* h);
}

struct b200m_pw {
    int device; uint32_t n_inst, bins, N; int f3, f4, f2; double rate;
    uint32_t rboff, smps, sps, step;                       // shared ring offset + 25 Hz analysis clock (gui/fft.c:43-64)
    int mode = 0;                                          // 0: phasewheel process_audio, 1: stereoscope process_audio
    float *d_ring = nullptr, *d_win = nullptr, *d_raw = nullptr, *d_phase = nullptr, *d_level = nullptr, *d_peak = nullptr;
    float2* d_tw = nullptr;
    b200m_cor* cor = nullptr;                              // attached correlation bank (fused feed), not owned
    cudaStream_t own = nullptr; HostStage stage; bool last_host = false;
};

static cudaStream_t pw_stream (b200m_pw* h, void* stream) { return h->last_host ? h->own : (cudaStream_t)stream; }
static size_t pw_smem_bytes (uint32_t N) { return (size_t)12 * N; }   // 2 x N/2 float2 + 2 x N/2 float

static int pw_process (b200m_pw* h, const float* d_in, size_t stride, uint32_t nfram, float db_thresh, int* fired, cudaStream_t st)
{
    // fftx_run walks the block in steps of at most window_size (gui/fft.c:346-360) and process_audio runs ONCE
    // after both channels' fftx_run (gui/phasewheel.c:1310-1313): when several analyses fire inside one call only
    // the last one's spectra survive, so only that one is launched (its ring state is the one at its firing time
    // because launches execute in stream order).
    int any = 0, last_fire = -1;
    {
        uint32_t sm = h->smps, d = 0; int step = 0;
        while (d < nfram) { const uint32_t n = (nfram - d) < h->N ? (nfram - d) : h->N; sm += n; if (sm >= h->sps) { sm = 0; last_fire = step; } d += n; ++step; }
    }
    // fused feed: the correlation kernel stages the block in shared memory anyway and appends it to the ring from there.  A block
    // longer than the window is walked in window-sized steps below, but Stcorrdsp::process must see it as ONE call (its scrub and
    // bias act per call, stcorrdsp.cc:65-75): such blocks run the correlation unfused, once, ahead of the steps.
    const bool fuse = h->cor && nfram <= h->N;
    if (h->cor && !fuse) { if (int rc = cor_feed (h->cor, d_in, stride, nfram, st, nullptr, 0, 0)) return rc; }
    uint32_t done = 0; int step = 0;
    while (done < nfram) {
        const uint32_t n = (nfram - done) < h->N ? (nfram - done) : h->N;
        if (fuse) {
            if (int rc = cor_feed (h->cor, d_in + done, stride, n, st, h->d_ring, (int)h->N, (int)h->rboff)) return rc;
        } else {
            const size_t total = (size_t)h->n_inst * 2 * n;
            pw_append_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>> (d_in + done, stride, (int)(h->n_inst * 2), (int)n, (int)h->N, (int)h->rboff, h->d_ring);
            B200M_LAUNCHED (1);
        }
        h->rboff = (h->rboff + n) % h->N;
        h->smps += n;
        if (h->smps >= h->sps) {                            // :308-313
            h->step = h->smps; h->smps = 0;
            if (step == last_fire) {
                pw_analyze_kernel<<<h->n_inst, PW_THREADS, pw_smem_bytes (h->N), st>>> (
                    h->d_ring, (int)h->N, h->f3, h->f4, h->f2, (int)h->rboff, h->d_win, h->d_tw, db_thresh, h->d_raw, h->d_phase, h->d_level, h->d_peak, h->mode);
                B200M_LAUNCHED (1);
            }
            any = 1;
        }
        done += n; ++step;
    }
    if (fired) *fired = any;
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

extern "C" {

int b200m_pw_create (b200m_pw** out, int device, uint32_t n_inst, uint32_t fft_bins, double rate)
{
    if (!out) return set_err (B200M_E_INVAL, "NULL out pointer");
    *out = nullptr;
    if (n_inst == 0 || !(rate >= 1000.0)) return set_err (B200M_E_INVAL, "bad n_inst/rate");
    // the sizes of the reference GUI's selector (gui/phasewheel.c:1108-1116): powers of two 64 .. 8192, and 6144
    if (fft_bins < 64 || fft_bins > 8192 || ((fft_bins & (fft_bins - 1)) && fft_bins != 6144)) return set_err (B200M_E_INVAL, "fft_bins must be a power of two in 64..8192, or 6144");
    if (b200m_device_count () <= 0) return set_err (B200M_E_NODEVICE, "no CUDA device: b200meters has no CPU path");
    DeviceGuard g (device);
    if (!g.ok) return set_err (B200M_E_NODEVICE, "cannot select CUDA device %d", device);
    b200m_pw* h = new (std::nothrow) b200m_pw;
    if (!h) return set_err (B200M_E_NOMEM, "host allocation failed");
    h->device = device; h->n_inst = n_inst; h->bins = fft_bins; h->N = 2 * fft_bins; h->rate = rate;
    {   // factor the complex transform length M = N / 2 = fft_bins into radix-3 / radix-4 / radix-2 passes
        uint32_t m = fft_bins; h->f3 = h->f4 = h->f2 = 0;
        while (m % 3 == 0) { ++h->f3; m /= 3; }
        while (m % 4 == 0) { ++h->f4; m /= 4; }
        while (m % 2 == 0) { ++h->f2; m /= 2; }
    }
    h->rboff = h->smps = h->step = 0;
    h->sps = (uint32_t)ceil (rate / 25);                    // fftx_init (..., rate, 25): gui/fft.c:219, phasewheel.c:193
    const uint32_t N = h->N;
    float* win = (float*)malloc (N * sizeof (float));
    float2* tw = (float2*)malloc (N * sizeof (float2));
    if (!win || !tw) { free (win); free (tw); delete h; return set_err (B200M_E_NOMEM, "host allocation failed"); }
    {   // Hann window, normalised to sum 2 (ft_hannhamm + ft_gen_window, gui/fft.c:69-79,122-161)
        double sum = 0.0; const double c = 2.0 * M_PI / (N - 1.0);
        for (uint32_t i = 0; i < N; ++i) { win[i] = .5 - .5 * cos (c * i); sum += win[i]; }
        const double isum = 2.0 / sum;
        for (uint32_t i = 0; i < N; ++i) win[i] *= isum;
    }
    for (uint32_t k = 0; k < N; ++k) { const double a = -2.0 * M_PI * (double)k / (double)N; tw[k] = make_float2 ((float)cos (a), (float)sin (a)); }
    cudaError_t e = cudaSuccess;
    auto A = [&] (void** p, size_t bytes) { if (e == cudaSuccess) { e = cudaMalloc (p, bytes); if (e == cudaSuccess) e = cudaMemset (*p, 0, bytes); } };
    A ((void**)&h->d_ring, (size_t)n_inst * 2 * N * sizeof (float));
    A ((void**)&h->d_win, N * sizeof (float));
    A ((void**)&h->d_tw, N * sizeof (float2));
    A ((void**)&h->d_phase, (size_t)n_inst * fft_bins * sizeof (float));
    A ((void**)&h->d_level, (size_t)n_inst * fft_bins * sizeof (float));
    A ((void**)&h->d_peak, n_inst * sizeof (float));
    if (e == cudaSuccess) e = cudaMemcpy (h->d_win, win, N * sizeof (float), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy (h->d_tw, tw, N * sizeof (float2), cudaMemcpyHostToDevice);
    free (win); free (tw);
    if (e == cudaSuccess) e = cudaFuncSetAttribute (pw_analyze_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pw_smem_bytes (16384));
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags (&h->own, cudaStreamNonBlocking);
    if (e == cudaSuccess) {
        const size_t n = (size_t)n_inst * fft_bins;       // ui->level[i] = -100, ui->phase[i] = 0 (phasewheel.c:199-202)
        pw_init_kernel<<<(unsigned)((n + 255) / 256), 256>>> (n, h->d_level, h->d_phase, 0.0f);
        B200M_LAUNCHED (1);
        e = cudaDeviceSynchronize ();
    }
    if (e != cudaSuccess) { int rc = cuda_fail (e, "pw_create", __FILE__, __LINE__); b200m_pw_destroy (h); return rc; }
    *out = h;
    return 0;
}

int b200m_pw_destroy (b200m_pw* h)
{
    if (!h) return 0;
    DeviceGuard g (h->device);
    cudaDeviceSynchronize ();
    cudaFree (h->d_ring); cudaFree (h->d_win); cudaFree (h->d_tw); cudaFree (h->d_raw); cudaFree (h->d_phase); cudaFree (h->d_level); cudaFree (h->d_peak);
    h->stage.release ();
    if (h->own) cudaStreamDestroy (h->own);
    delete h;
    return 0;
}

int b200m_pw_set_mode (b200m_pw* h, int mode)
{
    // selects which GUI's process_audio follows the two FFTs and re-initialises the outputs as that GUI's reinitialize_fft
    // does: phasewheel phase = 0 / level = -100 (gui/phasewheel.c:199-202), stereoscope lr = 0.5 / level = -100 (gui/stereoscope.c:143-146)
    if (!h || (mode != B200M_PW_PHASEWHEEL && mode != B200M_PW_STEREOSCOPE)) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    B200M_CUDA (cudaDeviceSynchronize ());
    h->mode = mode;
    const size_t n = (size_t)h->n_inst * h->bins;
    pw_init_kernel<<<(unsigned)((n + 255) / 256), 256>>> (n, h->d_level, h->d_phase, mode == B200M_PW_STEREOSCOPE ? 0.5f : 0.0f);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaMemset (h->d_peak, 0, h->n_inst * sizeof (float)));
    B200M_CUDA (cudaDeviceSynchronize ());
    return 0;
}

int b200m_pw_process_device (b200m_pw* h, const float* d_in, size_t stride, uint32_t nfram, float db_thresh, int* fired, void* stream)
{
    if (int rc = check_block_args (h, d_in, stride, nfram)) return rc;
    DeviceGuard g (h->device);
    h->last_host = false;
    return pw_process (h, d_in, stride, nfram, db_thresh, fired, (cudaStream_t)stream);
}

int b200m_pw_process_host (b200m_pw* h, const float* in, size_t stride, uint32_t nfram, float db_thresh, int* fired)
{
    if (int rc = check_block_args (h, in, stride, nfram)) return rc;
    DeviceGuard g (h->device);
    B200M_ENTER_HOST_PATH (h);
    if (h->stage.ensure ((size_t)2 * h->n_inst, nfram)) return set_err (B200M_E_NOMEM, "staging buffer allocation failed");
    B200M_CUDA (cudaMemcpy2DAsync (h->stage.d, h->stage.cap * sizeof (float), in, stride * sizeof (float),
                                   (size_t)nfram * sizeof (float), (size_t)2 * h->n_inst, cudaMemcpyHostToDevice, h->own));
    h->last_host = true;
    return pw_process (h, h->stage.d, h->stage.cap, nfram, db_thresh, fired, h->own);
}

int b200m_pw_results (b200m_pw* h, float* phase, float* level, float* peak, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    DeviceGuard g (h->device);
    cudaStream_t st = pw_stream (h, stream);
    const size_t nb = (size_t)h->n_inst * h->bins * sizeof (float);
    if (phase) B200M_CUDA (cudaMemcpyAsync (phase, h->d_phase, nb, cudaMemcpyDeviceToHost, st));
    if (level) B200M_CUDA (cudaMemcpyAsync (level, h->d_level, nb, cudaMemcpyDeviceToHost, st));
    if (peak)  B200M_CUDA (cudaMemcpyAsync (peak, h->d_peak, h->n_inst * sizeof (float), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_pw_debug_capture (b200m_pw* h, int enable)
{
    // the per-channel power / phase planes (ft->power, ft->phase) are intermediate results: 16 bytes per bin and analysis that only
    // tests read back, so they are written only while capture is on
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    DeviceGuard g (h->device);
    B200M_CUDA (cudaDeviceSynchronize ());
    if (enable && !h->d_raw) {
        B200M_CUDA (cudaMalloc ((void**)&h->d_raw, (size_t)h->n_inst * 4 * h->bins * sizeof (float)));
        B200M_CUDA (cudaMemset (h->d_raw, 0, (size_t)h->n_inst * 4 * h->bins * sizeof (float)));
    }
    if (!enable && h->d_raw) { cudaFree (h->d_raw); h->d_raw = nullptr; }
    return 0;
}

int b200m_pw_attach_cor (b200m_pw* h, b200m_cor* cor)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    if (cor && cor_instances (cor) != h->n_inst) return set_err (B200M_E_INVAL, "the correlation bank must have as many pairs as the phasewheel bank has instances");
    DeviceGuard g (h->device);
    B200M_CUDA (cudaDeviceSynchronize ());
    h->cor = cor;
    return 0;
}

int b200m_pw_raw (b200m_pw* h, uint32_t inst, float* powL, float* powR, float* phL, float* phR, void* stream)
{
    if (!h || inst >= h->n_inst) return set_err (B200M_E_INVAL, "bad argument");
    if (!h->d_raw) return set_err (B200M_E_INVAL, "raw spectra are only kept after b200m_pw_debug_capture (h, 1)");
    DeviceGuard g (h->device);
    cudaStream_t st = pw_stream (h, stream);
    float* dst[4] = {powL, powR, phL, phR};
    for (int q = 0; q < 4; ++q)
        if (dst[q]) B200M_CUDA (cudaMemcpyAsync (dst[q], h->d_raw + ((size_t)inst * 4 + q) * h->bins, h->bins * sizeof (float), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_pw_device_results (b200m_pw* h, const float** d_phase, const float** d_level, const float** d_peak)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    if (d_phase) *d_phase = h->d_phase;
    if (d_level) *d_level = h->d_level;
    if (d_peak) *d_peak = h->d_peak;
    return 0;
}

}  // extern "C"
