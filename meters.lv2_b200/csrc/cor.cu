// cor.cu — stereo phase-correlation bank.
//
// Replaces LV2M::Stcorrdsp (jmeters/stcorrdsp.cc:47-93) for N stereo pairs: five coupled one-pole
// recurrences per pair, strictly serial in time.  One lane owns one pair; a warp stages
// [32 pairs x 2 channels x 32 samples] tiles in shared memory with a 4-deep cp.async pipeline
// (separate L and R planes, row pitch 36 floats so that LDS.128 by 32 lanes is conflict free).
// Operation order is the reference's, without FMA contraction (bit-identical state).
#include <math.h>
#include <stdlib.h>
#include <vector>
#include "common.cuh"

namespace b200m {

constexpr int COR_T = 32, COR_P = COR_T + 4, COR_STAGES = 4;

// HOLD (b200m_cor_process_ctl_*): pairs with run[i] == 0 are held -- their rows are never loaded and their state and reading are
// not written back.  The plain process calls and the phasewheel ring feed are the HOLD = false instantiation.
template <bool HOLD>
__global__ void __launch_bounds__ (32)
cor_kernel (const float* __restrict__ in, size_t stride, int n_inst, int nfram, int aligned, float w1, float w2,
            float* __restrict__ st /* [5][n_inst] */, float* __restrict__ res, float* __restrict__ ring, int N, int rboff,
            const uint8_t* __restrict__ run)
{
    __shared__ __align__ (16) float tile[COR_STAGES][2][32 * COR_P];
    const int lane = threadIdx.x;
    const int i0 = blockIdx.x * 32;
    const int inst = min (i0 + lane, n_inst - 1);
    const bool live = (i0 + lane) < n_inst;
    const int ntiles = (nfram + COR_T - 1) / COR_T;
    // bit p: pair i0 + p is held (lanes past the bank repeat its last pair); a warp of held pairs has nothing to do
    const unsigned held = HOLD ? __ballot_sync (0xffffffffu, !run[inst]) : 0u;
    if (HOLD && held == 0xffffffffu) return;

    auto issue = [&] (int t) {
        if (t < ntiles) {
            const int s0 = t * COR_T;
            float* d0 = tile[t % COR_STAGES][0];
            if (aligned) {
                const int c4 = (lane & 7) * 4;
                const int left = (nfram - (s0 + c4)) * 4;
                const int nb = left >= 16 ? 16 : (left > 0 ? left : 0);
#pragma unroll
                for (int i = 0; i < 16; ++i) {                 // 64 rows, 4 rows per instruction
                    const int row = 4 * i + (lane >> 3);       // 0..63 : pair = row>>1, channel = row&1
                    const int pr = min (i0 + (row >> 1), n_inst - 1);
                    const float* src = in + (size_t)(2 * pr + (row & 1)) * stride + s0 + c4;
                    const int nr = (held >> (row >> 1)) & 1 ? 0 : nb;
                    cp_async16 (d0 + (row & 1) * (32 * COR_P) + (row >> 1) * COR_P + c4, nr ? src : in, nr);
                }
            } else {
#pragma unroll 4
                for (int row = 0; row < 64; ++row) {
                    const int pr = min (i0 + (row >> 1), n_inst - 1);
                    const bool ok = (s0 + lane) < nfram && !((held >> (row >> 1)) & 1);
                    cp_async4 (d0 + (row & 1) * (32 * COR_P) + (row >> 1) * COR_P + lane,
                               ok ? in + (size_t)(2 * pr + (row & 1)) * stride + s0 + lane : in, ok ? 4 : 0);
                }
            }
        }
        cp_async_commit ();
    };

    float zl = st[0 * (size_t)n_inst + inst], zr = st[1 * (size_t)n_inst + inst];
    float zlr = st[2 * (size_t)n_inst + inst], zll = st[3 * (size_t)n_inst + inst], zrr = st[4 * (size_t)n_inst + inst];

    auto step = [&] (float l, float r) {                         // stcorrdsp.cc:58-62
        zl = __fadd_rn (zl, __fadd_rn (__fmul_rn (w1, __fsub_rn (l, zl)), 1e-20f));
        zr = __fadd_rn (zr, __fadd_rn (__fmul_rn (w1, __fsub_rn (r, zr)), 1e-20f));
        zlr = __fadd_rn (zlr, __fmul_rn (w2, __fsub_rn (__fmul_rn (zl, zr), zlr)));
        zll = __fadd_rn (zll, __fmul_rn (w2, __fsub_rn (__fmul_rn (zl, zl), zll)));
        zrr = __fadd_rn (zrr, __fmul_rn (w2, __fsub_rn (__fmul_rn (zr, zr), zrr)));
    };

#pragma unroll
    for (int t = 0; t < COR_STAGES - 1; ++t) issue (t);
    for (int t = 0; t < ntiles; ++t) {
        cp_async_wait<COR_STAGES - 2> ();
        __syncwarp ();
        const float* pl = tile[t % COR_STAGES][0] + lane * COR_P;
        const float* pr = tile[t % COR_STAGES][1] + lane * COR_P;
        const int len = min (COR_T, nfram - t * COR_T);
        if (!HOLD && ring && lane < len) {
            // fused phasewheel feed (b200m_pw_attach_cor): r_buf[(i + n_off) % n_siz] = data[i] (gui/fft.c:302-305) for the 64 rows
            // of this tile, one 128-byte row segment per store instruction
            int o = rboff + t * COR_T + lane; if (o >= N) o -= N;
            const int rows = min (32, n_inst - i0);
            for (int pr_ = 0; pr_ < rows; ++pr_) {
                ring[((size_t)(i0 + pr_) * 2 + 0) * N + o] = tile[t % COR_STAGES][0][pr_ * COR_P + lane];
                ring[((size_t)(i0 + pr_) * 2 + 1) * N + o] = tile[t % COR_STAGES][1][pr_ * COR_P + lane];
            }
        }
        int j = 0;
        for (; j + 4 <= len; j += 4) {
            const float4 a = *reinterpret_cast<const float4*> (pl + j);
            const float4 b = *reinterpret_cast<const float4*> (pr + j);
            step (a.x, b.x); step (a.y, b.y); step (a.z, b.z); step (a.w, b.w);
        }
        for (; j < len; ++j) step (pl[j], pr[j]);
        __syncwarp ();
        issue (t + COR_STAGES - 1);
    }
    cp_async_wait<0> ();
    // end of process(): non-finite scrub, anti-denormal bias on the three products (:65-75)
    zl = scrub (zl); zr = scrub (zr); zlr = scrub (zlr); zll = scrub (zll); zrr = scrub (zrr);
    zlr = __fadd_rn (zlr, 1e-10f); zll = __fadd_rn (zll, 1e-10f); zrr = __fadd_rn (zrr, 1e-10f);
    if (live && !((held >> lane) & 1)) {
        st[0 * (size_t)n_inst + inst] = zl;  st[1 * (size_t)n_inst + inst] = zr;
        st[2 * (size_t)n_inst + inst] = zlr; st[3 * (size_t)n_inst + inst] = zll; st[4 * (size_t)n_inst + inst] = zrr;
        // Stcorrdsp::read (:79-82)
        res[inst] = __fdiv_rn (zlr, __fsqrt_rn (__fadd_rn (__fmul_rn (zll, zrr), 1e-10f)));
    }
}

// ---- time-parallel evaluation (B200M_PREC_FMA) ---------------------------------------------------------------------------
// Stcorrdsp's recurrences (stcorrdsp.cc:58-62) are one-pole filters, i.e. affine maps of their state:
//   zl' = (1 - w1) zl + (w1 l + 1e-20),   zlr' = (1 - w2) zlr + w2 (zl' zr')   (zr, zll, zrr alike),
// and affine maps compose: one warp owns ONE pair, lane j takes frames [32 j, 32 j + 32) of a 1024-frame superchunk,
//   pass 1: zl, zr over the own segment from a zero state           -> (A, B) with  end = A * start + B,  A = (1 - w1)^count
//   warp scan (Hillis-Steele on the (A, B) pairs)                    -> the true state at the start of every segment
//   pass 2: zl, zr again from the true start state, the three product filters from zero, same scan for their block-end state.
// The per-sample operations are the reference's; only the stitching differs (rounding at the 1e-7 level, contract 1e-5).
// A bank of 2048 pairs is 2048 warps instead of the 64 of cor_kernel, and 256 pairs per GPU (C5 over eight GPUs) still fill a chip.
constexpr int CSC_WARPS = 4, CSC_SEG = 32, CSC_SUPER = 32 * CSC_SEG, CSC_PITCH = CSC_SEG + 1;

// the product filters forget over 1 / w2 = 14400 samples: their composite multiplier (1 - w2)^n is carried in double, because
// fl (1 - w2) is off by up to 3e-8 and that error would compound to 4e-4 over the filter's memory
B200M_DEV void affine_scan_d (double& A, double& B, int lane)
{
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const double Ap = __shfl_up_sync (0xffffffffu, A, d), Bp = __shfl_up_sync (0xffffffffu, B, d);
        if (lane >= d) { B = __fma_rn (A, Bp, B); A = __dmul_rn (A, Ap); }
    }
}

B200M_DEV void affine_scan (float& A, float& B, int lane)
{
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const float Ap = __shfl_up_sync (0xffffffffu, A, d), Bp = __shfl_up_sync (0xffffffffu, B, d);
        if (lane >= d) { B = fmaf (A, Bp, B); A = A * Ap; }
    }
}

template <bool HOLD>
__global__ void __launch_bounds__ (CSC_WARPS * 32)
cor_scan_kernel (const float* __restrict__ in, size_t stride, int n_inst, int nfram, int aligned, float w1, float w2,
                 float* __restrict__ st /* [5][n_inst] */, float* __restrict__ res, float* __restrict__ ring, int N, int rboff,
                 const uint8_t* __restrict__ run)
{
    __shared__ float sm[CSC_WARPS][2][32 * CSC_PITCH];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int inst = blockIdx.x * CSC_WARPS + warp;
    if (inst >= n_inst || (HOLD && !run[inst])) return;      // warp-uniform; warps never synchronise with each other
    if (HOLD) ring = nullptr;                                // the phasewheel ring feed never holds: compiled out of this variant
    float* sl = sm[warp][0]; float* sr = sm[warp][1];
    const float* gl = in + (size_t)(2 * inst) * stride; const float* gr = gl + stride;
    float* rl = ring ? ring + (size_t)(2 * inst) * N : nullptr; float* rr = rl ? rl + N : nullptr;
    const bool ring4 = aligned && (N % 4 == 0) && (rboff % 4 == 0);
    float zl = st[0 * (size_t)n_inst + inst], zr = st[1 * (size_t)n_inst + inst];
    float zlr = st[2 * (size_t)n_inst + inst], zll = st[3 * (size_t)n_inst + inst], zrr = st[4 * (size_t)n_inst + inst];
    const float a1 = 1.0f - w1;
    const double a2 = 1.0 - (double)w2;                      // exact

    for (int s0 = 0; s0 < nfram; s0 += CSC_SUPER) {
        const int len = min (CSC_SUPER, nfram - s0);
        __syncwarp ();
        // stage the superchunk: frame f of the chunk -> slot (f / 32) * 33 + f % 32 (lane j then walks its own 33-float row)
        if (aligned) {
            // all sixteen 16-byte loads of the superchunk are issued before the first one is used (32 KB in flight per CTA)
            float4 vl[CSC_SUPER / 128], vr[CSC_SUPER / 128];
#pragma unroll
            for (int i = 0; i < CSC_SUPER / 128; ++i) {
                const int f = 4 * (i * 32 + lane);
                vl[i] = make_float4 (0.f, 0.f, 0.f, 0.f); vr[i] = vl[i];
                if (f + 4 <= len) { vl[i] = *reinterpret_cast<const float4*> (gl + s0 + f); vr[i] = *reinterpret_cast<const float4*> (gr + s0 + f); }
                else if (f < len) {                            // the last group of a ragged block: 1..3 valid samples
                    vl[i] = make_float4 (gl[s0 + f], f + 1 < len ? gl[s0 + f + 1] : 0.f, f + 2 < len ? gl[s0 + f + 2] : 0.f, 0.f);
                    vr[i] = make_float4 (gr[s0 + f], f + 1 < len ? gr[s0 + f + 1] : 0.f, f + 2 < len ? gr[s0 + f + 2] : 0.f, 0.f);
                }
            }
#pragma unroll
            for (int i = 0; i < CSC_SUPER / 128; ++i) {
                const int f = 4 * (i * 32 + lane);
                if (f < len) {
                    const int slot = (f >> 5) * CSC_PITCH + (f & 31);
                    sl[slot] = vl[i].x; sl[slot + 1] = vl[i].y; sl[slot + 2] = vl[i].z; sl[slot + 3] = vl[i].w;
                    sr[slot] = vr[i].x; sr[slot + 1] = vr[i].y; sr[slot + 2] = vr[i].z; sr[slot + 3] = vr[i].w;
                    if (rl) {
                        int o = rboff + s0 + f; o %= N;
                        if (ring4 && f + 4 <= len) { *reinterpret_cast<float4*> (rl + o) = vl[i]; *reinterpret_cast<float4*> (rr + o) = vr[i]; }
                        else {
                            const float al[4] = {vl[i].x, vl[i].y, vl[i].z, vl[i].w}, ar[4] = {vr[i].x, vr[i].y, vr[i].z, vr[i].w};
                            for (int c = 0; c < 4 && f + c < len; ++c) { int oc = o + c; if (oc >= N) oc -= N; rl[oc] = al[c]; rr[oc] = ar[c]; }
                        }
                    }
                }
            }
        } else {
            for (int i = 0; i < CSC_SEG; ++i) {
                const int f = i * 32 + lane;
                if (f < len) {
                    const float vl = gl[s0 + f], vr = gr[s0 + f];
                    sl[i * CSC_PITCH + lane] = vl; sr[i * CSC_PITCH + lane] = vr;
                    if (rl) { const int o = (rboff + s0 + f) % N; rl[o] = vl; rr[o] = vr; }
                }
            }
        }
        __syncwarp ();
        const int cnt = max (0, min (CSC_SEG, len - lane * CSC_SEG));
        const float* pl = sl + lane * CSC_PITCH; const float* pr = sr + lane * CSC_PITCH;
        // pass 1: zl, zr of the own segment from a zero state
        float A = 1.0f, el = 0.0f, er = 0.0f;
        for (int i = 0; i < cnt; ++i) {
            el = __fadd_rn (el, __fadd_rn (__fmul_rn (w1, __fsub_rn (pl[i], el)), 1e-20f));
            er = __fadd_rn (er, __fadd_rn (__fmul_rn (w1, __fsub_rn (pr[i], er)), 1e-20f));
            A *= a1;
        }
        float Al = A, Ar = A;
        affine_scan (Al, el, lane); affine_scan (Ar, er, lane);             // (Al, el): composite of segments 0 .. lane
        const float endl = fmaf (Al, zl, el), endr = fmaf (Ar, zr, er);       // state at the END of this lane's segment
        float sl0 = __shfl_up_sync (0xffffffffu, endl, 1), sr0 = __shfl_up_sync (0xffffffffu, endr, 1);
        if (lane == 0) { sl0 = zl; sr0 = zr; }
        // pass 2: from the true start state; the product filters from zero
        float xl = sl0, xr = sr0, plr = 0.0f, pll = 0.0f, prr = 0.0f; double Bq = 1.0;
        for (int i = 0; i < cnt; ++i) {
            xl = __fadd_rn (xl, __fadd_rn (__fmul_rn (w1, __fsub_rn (pl[i], xl)), 1e-20f));
            xr = __fadd_rn (xr, __fadd_rn (__fmul_rn (w1, __fsub_rn (pr[i], xr)), 1e-20f));
            plr = __fadd_rn (plr, __fmul_rn (w2, __fsub_rn (__fmul_rn (xl, xr), plr)));
            pll = __fadd_rn (pll, __fmul_rn (w2, __fsub_rn (__fmul_rn (xl, xl), pll)));
            prr = __fadd_rn (prr, __fmul_rn (w2, __fsub_rn (__fmul_rn (xr, xr), prr)));
            Bq = __dmul_rn (Bq, a2);
        }
        double B1 = Bq, B2 = Bq, B3 = Bq, dlr = plr, dll = pll, drr = prr;
        affine_scan_d (B1, dlr, lane); affine_scan_d (B2, dll, lane); affine_scan_d (B3, drr, lane);
        // block-end state = the composite of all 32 segments (lane 31) applied to the previous state
        zlr = __shfl_sync (0xffffffffu, __double2float_rn (__fma_rn (B1, (double)zlr, dlr)), 31);
        zll = __shfl_sync (0xffffffffu, __double2float_rn (__fma_rn (B2, (double)zll, dll)), 31);
        zrr = __shfl_sync (0xffffffffu, __double2float_rn (__fma_rn (B3, (double)zrr, drr)), 31);
        zl = __shfl_sync (0xffffffffu, endl, 31); zr = __shfl_sync (0xffffffffu, endr, 31);
    }
    // end of process(): non-finite scrub, anti-denormal bias on the three products (:65-75)
    zl = scrub (zl); zr = scrub (zr); zlr = scrub (zlr); zll = scrub (zll); zrr = scrub (zrr);
    zlr = __fadd_rn (zlr, 1e-10f); zll = __fadd_rn (zll, 1e-10f); zrr = __fadd_rn (zrr, 1e-10f);
    if (lane == 0) {
        st[0 * (size_t)n_inst + inst] = zl;  st[1 * (size_t)n_inst + inst] = zr;
        st[2 * (size_t)n_inst + inst] = zlr; st[3 * (size_t)n_inst + inst] = zll; st[4 * (size_t)n_inst + inst] = zrr;
        res[inst] = __fdiv_rn (zlr, __fsqrt_rn (__fadd_rn (__fmul_rn (zll, zrr), 1e-10f)));          // Stcorrdsp::read (:79-82)
    }
}

// pairs [i0, i0 + n) back to a newly constructed Stcorrdsp (stcorrdsp.cc:33-37): the five filter states and the reading zero
__global__ void cor_clear_kernel (int n_inst, int i0, int n, float* __restrict__ st, float* __restrict__ res)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
#pragma unroll
    for (int q = 0; q < 5; ++q) st[q * (size_t)n_inst + i0 + i] = 0.0f;
    res[i0 + i] = 0.0f;
}

}  // namespace b200m

using namespace b200m;

struct b200m_cor {
    int device; uint32_t n_inst; float w1, w2;
    int scan = 0;                          // B200M_PREC_FMA: time-parallel cor_scan_kernel
    float *d_st = nullptr, *d_res = nullptr;
    std::vector<uint8_t> run;              // b200m_cor_process_ctl_*: the run mask as last uploaded to d_run (all 1 at create)
    uint8_t* d_run = nullptr;
    cudaStream_t own = nullptr; HostStage stage; bool last_host = false;
};

static cudaStream_t cor_stream (b200m_cor* h, void* stream) { return h->last_host ? h->own : (cudaStream_t)stream; }

template <bool HOLD>
static int cor_launch (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, cudaStream_t st, float* ring, int N, int rboff)
{
    const int aligned = ((uintptr_t)d_in % 16 == 0) && (stride % 4 == 0);
    const uint8_t* run = HOLD ? h->d_run : nullptr;
    if (h->scan)
        cor_scan_kernel<HOLD><<<(h->n_inst + CSC_WARPS - 1) / CSC_WARPS, CSC_WARPS * 32, 0, st>>> (
            d_in, stride, (int)h->n_inst, (int)nfram, aligned, h->w1, h->w2, h->d_st, h->d_res, ring, N, rboff, run);
    else
        cor_kernel<HOLD><<<(h->n_inst + 31) / 32, 32, 0, st>>> (d_in, stride, (int)h->n_inst, (int)nfram, aligned, h->w1, h->w2, h->d_st, h->d_res,
                                                                ring, N, rboff, run);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

namespace b200m {
int cor_feed (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, cudaStream_t st, float* ring, int N, int rboff)
{
    return cor_launch<false> (h, d_in, stride, nfram, st, ring, N, rboff);
}
uint32_t cor_instances (const b200m_cor* h) { return h ? h->n_inst : 0; }
}

// run: NULL (every pair runs) or n_inst flags; the mask is uploaded only when it differs from the last one
static int cor_process (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, const uint8_t* run, cudaStream_t st)
{
    if (!run) return cor_launch<false> (h, d_in, stride, nfram, st, nullptr, 0, 0);
    if (memcmp (run, h->run.data (), h->n_inst)) {
        for (uint32_t i = 0; i < h->n_inst; ++i) h->run[i] = run[i] != 0;
        B200M_CUDA (cudaMemcpyAsync (h->d_run, h->run.data (), h->n_inst, cudaMemcpyHostToDevice, st));
    }
    return cor_launch<true> (h, d_in, stride, nfram, st, nullptr, 0, 0);
}

extern "C" {

int b200m_design_cor (int fsamp, float flp, float tcf, float w[2])
{
    if (!w || fsamp < 1000) return set_err (B200M_E_INVAL, "bad argument");
    w[0] = 6.28f * flp / fsamp;                    // Stcorrdsp::init (stcorrdsp.cc:85-93), int fsamp
    w[1] = 1 / (tcf * fsamp);
    return 0;
}

int b200m_cor_create (b200m_cor** out, int device, uint32_t n_inst, int fsamp, float flp, float tcf)
{
    if (!out) return set_err (B200M_E_INVAL, "NULL out pointer");
    *out = nullptr;
    if (n_inst == 0 || fsamp < 1000) return set_err (B200M_E_INVAL, "bad n_inst/fsamp");
    if (b200m_device_count () <= 0) return set_err (B200M_E_NODEVICE, "no CUDA device: b200meters has no CPU path");
    DeviceGuard g (device);
    if (!g.ok) return set_err (B200M_E_NODEVICE, "cannot select CUDA device %d", device);
    b200m_cor* h = new (std::nothrow) b200m_cor;
    if (!h) return set_err (B200M_E_NOMEM, "host allocation failed");
    h->device = device; h->n_inst = n_inst;
    h->run.assign (n_inst, 1);
    { float w[2]; b200m_design_cor (fsamp, flp, tcf, w); h->w1 = w[0]; h->w2 = w[1]; }
    cudaError_t e = cudaMalloc ((void**)&h->d_st, (size_t)5 * n_inst * sizeof (float));
    if (e == cudaSuccess) e = cudaMemset (h->d_st, 0, (size_t)5 * n_inst * sizeof (float));
    if (e == cudaSuccess) e = cudaMalloc ((void**)&h->d_res, n_inst * sizeof (float));
    if (e == cudaSuccess) e = cudaMemset (h->d_res, 0, n_inst * sizeof (float));
    if (e == cudaSuccess) e = cudaMalloc ((void**)&h->d_run, n_inst);
    if (e == cudaSuccess) e = cudaMemset (h->d_run, 1, n_inst);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags (&h->own, cudaStreamNonBlocking);
    if (e != cudaSuccess) { int rc = cuda_fail (e, "cor_create", __FILE__, __LINE__); b200m_cor_destroy (h); return rc; }
    *out = h;
    return 0;
}

int b200m_cor_destroy (b200m_cor* h)
{
    if (!h) return 0;
    DeviceGuard g (h->device);
    cudaDeviceSynchronize ();
    cudaFree (h->d_st); cudaFree (h->d_res); cudaFree (h->d_run); h->stage.release ();
    if (h->own) cudaStreamDestroy (h->own);
    delete h;
    return 0;
}

int b200m_cor_process_ctl_device (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, const uint8_t* run, void* stream)
{
    if (int rc = check_block_args (h, d_in, stride, nfram)) return rc;
    DeviceGuard g (h->device);
    h->last_host = false;
    return cor_process (h, d_in, stride, nfram, run, (cudaStream_t)stream);
}

int b200m_cor_process_device (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, void* stream)
{
    return b200m_cor_process_ctl_device (h, d_in, stride, nfram, nullptr, stream);
}

int b200m_cor_process_ctl_host (b200m_cor* h, const float* in, size_t stride, uint32_t nfram, const uint8_t* run)
{
    if (int rc = check_block_args (h, in, stride, nfram)) return rc;
    DeviceGuard g (h->device);
    B200M_ENTER_HOST_PATH (h);
    if (h->stage.ensure ((size_t)2 * h->n_inst, nfram)) return set_err (B200M_E_NOMEM, "staging buffer allocation failed");
    B200M_CUDA (cudaMemcpy2DAsync (h->stage.d, h->stage.cap * sizeof (float), in, stride * sizeof (float),
                                   (size_t)nfram * sizeof (float), (size_t)2 * h->n_inst, cudaMemcpyHostToDevice, h->own));
    h->last_host = true;
    return cor_process (h, h->stage.d, h->stage.cap, nfram, run, h->own);
}

int b200m_cor_process_host (b200m_cor* h, const float* in, size_t stride, uint32_t nfram)
{
    return b200m_cor_process_ctl_host (h, in, stride, nfram, nullptr);
}

int b200m_cor_set_precision (b200m_cor* h, int mode)
{
    if (!h || (mode != B200M_PREC_EXACT && mode != B200M_PREC_FMA)) return set_err (B200M_E_INVAL, "bad argument");
    h->scan = mode == B200M_PREC_FMA;                       // takes effect with the next process call
    return 0;
}

int b200m_cor_clear (b200m_cor* h, int32_t inst, void* stream)
{
    if (!h || inst < -1 || inst >= (int32_t)h->n_inst) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    const int i0 = inst < 0 ? 0 : inst, n = inst < 0 ? (int)h->n_inst : 1;
    cor_clear_kernel<<<(n + 127) / 128, 128, 0, cor_stream (h, stream)>>> ((int)h->n_inst, i0, n, h->d_st, h->d_res);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

int b200m_cor_results (b200m_cor* h, float* out, void* stream)
{
    if (!h || !out) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = cor_stream (h, stream);
    B200M_CUDA (cudaMemcpyAsync (out, h->d_res, h->n_inst * sizeof (float), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_cor_state (b200m_cor* h, float* state5, void* stream)
{
    if (!h || !state5) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = cor_stream (h, stream);
    const size_t n = h->n_inst;
    float* tmp = (float*)malloc (5 * n * sizeof (float));
    if (!tmp) return set_err (B200M_E_NOMEM, "host allocation failed");
    cudaError_t e = cudaMemcpyAsync (tmp, h->d_st, 5 * n * sizeof (float), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize (st);
    if (e != cudaSuccess) { free (tmp); return cuda_fail (e, "cor_state", __FILE__, __LINE__); }
    for (size_t i = 0; i < n; ++i) for (int q = 0; q < 5; ++q) state5[5 * i + q] = tmp[q * n + i];
    free (tmp);
    return 0;
}

int b200m_cor_coeffs (const b200m_cor* h, float w[2])
{
    if (!h || !w) return set_err (B200M_E_INVAL, "NULL argument");
    w[0] = h->w1; w[1] = h->w2;
    return 0;
}

}  // extern "C"
