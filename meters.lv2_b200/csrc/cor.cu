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

// RAG (b200m_cor_process_ragged_* and b200m_cor_process_ctl_*): pair i runs process() over its first rlen[i] <= nfram frames only.
// Each lane stops at its own end; the warp stages tiles up to its longest pair.  A pair with rlen[i] == 0 is not called (held): its
// rows are never loaded and its state and reading are not written back.  The plain process calls and the phasewheel ring feed are
// the RAG = false instantiation.
// HIST (b200m_cor_hist_enable): after each frame's five updates the lane also forms the frame's reading r (Stcorrdsp::read, :79-82,
// on the in-loop state) and, if zll + zrr >= thr and r is finite, adds (double) r to the pair's fp64 sum in frame order and counts
// the frame in bin clamp (floor ((r + 1) * 100), 0, 199).  The counts are run-length coded in registers: the reading moves slowly
// (its filters smooth over tcf * fsamp frames), so a lane holds (bin, run) and adds the run to its own row of hcnt with one
// fire-and-forget atomic (RED) only when the bin changes and at kernel end.  The recurrences, states and readings are the same bits
// as without the plane; the per-frame reading's cost is in DESIGN.md §3.
template <bool RAG, bool HIST = false>
__global__ void __launch_bounds__ (32)
cor_kernel (const float* __restrict__ in, size_t stride, int n_inst, int nfram, int aligned, float w1, float w2,
            float* __restrict__ st /* [5][n_inst] */, float* __restrict__ res, float* __restrict__ ring, int N, int rboff,
            const uint32_t* __restrict__ rlen, unsigned long long* __restrict__ hcnt /* [n_inst][200] */,
            double* __restrict__ hsum /* [n_inst] */, float thr)
{
    __shared__ __align__ (16) float tile[COR_STAGES][2][32 * COR_P];
    const int lane = threadIdx.x;
    const int i0 = blockIdx.x * 32;
    const int inst = min (i0 + lane, n_inst - 1);
    const bool live = (i0 + lane) < n_inst;
    const int rl = RAG ? (int)rlen[inst] : nfram;          // this pair's end
    const int wend = RAG ? __reduce_max_sync (0xffffffffu, rl) : nfram;
    const int ntiles = (wend + COR_T - 1) / COR_T;
    // bit p: pair i0 + p is held (lanes past the bank repeat its last pair); a warp of held pairs has nothing to do
    const unsigned held = RAG ? __ballot_sync (0xffffffffu, rl == 0) : 0u;
    if (RAG && held == 0xffffffffu) return;

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

    double hs = 0.0; int hbin = 0; uint32_t hrun = 0;            // HIST: the pair's sum, and the open run of frames in bin hbin
    if constexpr (HIST) hs = hsum[inst];
    auto flush = [&] () {                                        // lanes past the bank repeat its last pair: they add nothing
        if (live && hrun) atomicAdd (hcnt + (size_t)inst * B200M_COR_HIST_BINS + hbin, (unsigned long long)hrun);
    };
    auto tally = [&] () {
        const float r = __fdiv_rn (zlr, __fsqrt_rn (__fadd_rn (__fmul_rn (zll, zrr), 1e-10f)));
        if (__fadd_rn (zll, zrr) >= thr && finitef_ (r)) {
            const int k = (int)fminf (fmaxf (floorf (__fmul_rn (__fadd_rn (r, 1.0f), 100.0f)), 0.0f), (float)(B200M_COR_HIST_BINS - 1));
            hs = __dadd_rn (hs, (double)r);
            if (k != hbin) { flush (); hbin = k; hrun = 0; }
            ++hrun;
        }
    };

#pragma unroll
    for (int t = 0; t < COR_STAGES - 1; ++t) issue (t);
    for (int t = 0; t < ntiles; ++t) {
        cp_async_wait<COR_STAGES - 2> ();
        __syncwarp ();
        const float* pl = tile[t % COR_STAGES][0] + lane * COR_P;
        const float* pr = tile[t % COR_STAGES][1] + lane * COR_P;
        const int len = min (COR_T, nfram - t * COR_T);
        if (!RAG && ring && lane < len) {
            // fused phasewheel feed (b200m_pw_attach_cor): r_buf[(i + n_off) % n_siz] = data[i] (gui/fft.c:302-305) for the 64 rows
            // of this tile, one 128-byte row segment per store instruction
            int o = rboff + t * COR_T + lane; if (o >= N) o -= N;
            const int rows = min (32, n_inst - i0);
            for (int pr_ = 0; pr_ < rows; ++pr_) {
                ring[((size_t)(i0 + pr_) * 2 + 0) * N + o] = tile[t % COR_STAGES][0][pr_ * COR_P + lane];
                ring[((size_t)(i0 + pr_) * 2 + 1) * N + o] = tile[t % COR_STAGES][1][pr_ * COR_P + lane];
            }
        }
        const int e = RAG ? max (0, min (COR_T, rl - t * COR_T)) : len;       // this pair's samples in the tile
        int j = 0;
        auto frame = [&] (float l, float r) {
            step (l, r);
            if constexpr (HIST) tally ();
        };
        for (; j + 4 <= e; j += 4) {
            const float4 a = *reinterpret_cast<const float4*> (pl + j);
            const float4 b = *reinterpret_cast<const float4*> (pr + j);
            frame (a.x, b.x); frame (a.y, b.y); frame (a.z, b.z); frame (a.w, b.w);
        }
        for (; j < e; ++j) frame (pl[j], pr[j]);
        __syncwarp ();
        issue (t + COR_STAGES - 1);
    }
    cp_async_wait<0> ();
    if constexpr (HIST) flush ();
    // end of process(): non-finite scrub, anti-denormal bias on the three products (:65-75)
    zl = scrub (zl); zr = scrub (zr); zlr = scrub (zlr); zll = scrub (zll); zrr = scrub (zrr);
    zlr = __fadd_rn (zlr, 1e-10f); zll = __fadd_rn (zll, 1e-10f); zrr = __fadd_rn (zrr, 1e-10f);
    if (live && rl > 0) {
        st[0 * (size_t)n_inst + inst] = zl;  st[1 * (size_t)n_inst + inst] = zr;
        st[2 * (size_t)n_inst + inst] = zlr; st[3 * (size_t)n_inst + inst] = zll; st[4 * (size_t)n_inst + inst] = zrr;
        // Stcorrdsp::read (:79-82)
        res[inst] = __fdiv_rn (zlr, __fsqrt_rn (__fadd_rn (__fmul_rn (zll, zrr), 1e-10f)));
        if constexpr (HIST) hsum[inst] = hs;
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

// RAG: pair inst runs over its first rlen[inst] frames, the warp's block length (warp-uniform: the segment layout is the same as for
// a plain block of that length); rlen 0: not called.
template <bool RAG>
__global__ void __launch_bounds__ (CSC_WARPS * 32)
cor_scan_kernel (const float* __restrict__ in, size_t stride, int n_inst, int nfram, int aligned, float w1, float w2,
                 float* __restrict__ st /* [5][n_inst] */, float* __restrict__ res, float* __restrict__ ring, int N, int rboff,
                 const uint32_t* __restrict__ rlen)
{
    __shared__ float sm[CSC_WARPS][2][32 * CSC_PITCH];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int inst = blockIdx.x * CSC_WARPS + warp;
    if (inst >= n_inst) return;                              // warp-uniform; warps never synchronise with each other
    if (RAG) {
        nfram = (int)rlen[inst];
        if (nfram == 0) return;
        ring = nullptr;                                      // the phasewheel ring feed is never ragged: compiled out of this variant
    }
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
    int scan = 0;                          // B200M_PREC_FMA: time-parallel cor_scan_kernel (when 1 / w2 <= COR_SCAN_MAX_MEMORY)
    float *d_st = nullptr, *d_res = nullptr;
    // ragged blocks (b200m_cor_process_ragged_*, and b200m_cor_process_ctl_* as lengths run[i] ? nfram : 0): the lengths as last
    // uploaded to rag.d (empty: none yet); a block uploads them only when they differ
    std::vector<uint32_t> len; RaggedLen rag;
    std::vector<uint32_t> ctl_len;         // b200m_cor_process_ctl_*: scratch for its lengths
    int attached = 0;                      // phasewheel banks feeding this one (b200m_pw_attach_cor): ragged calls are refused
    BankPath path;
    // the correlation histogram plane (b200m_cor_hist_enable): [n_inst][200] uint64 counts, then [n_inst] fp64 sums, in one allocation
    // so that a read is one copy; allocated on first use, kept until destroy
    void* d_hist = nullptr;
    bool hist = false;
    float hist_thr = 0.0f;                 // the gate on zll + zrr
    unsigned long long* hist_cnt () const { return (unsigned long long*)d_hist; }
    double* hist_sum () const { return (double*)(hist_cnt () + (size_t)n_inst * B200M_COR_HIST_BINS); }
    size_t hist_bytes () const { return (size_t)n_inst * (B200M_COR_HIST_BINS * sizeof (unsigned long long) + sizeof (double)); }
};

// The tolerance mode's promise is 1e-5 of the reference, and the reference's own fp32 rounding noise grows with the product filters'
// memory 1 / w2 = tcf * fs: the scan, ~1e-6 from float64 arithmetic, cannot track it beyond this many samples.  Measured on an H100
// (60 s per rate, tests/test_tolerance_rates_gpu.py): worst |scan - reference| <= 5.8e-6 up to 21600 samples (0.3 s up to 72 kHz,
// 0.45 s at 48 kHz), 8.3e-6 at 26460 (88.2 kHz), 1.5e-5 at 52920 (176.4 kHz).  A longer memory runs cor_kernel, bit-identical.
constexpr float COR_SCAN_MAX_MEMORY = 21600.0f;

template <bool RAG>
static int cor_launch (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, cudaStream_t st, float* ring, int N, int rboff)
{
    const int aligned = ((uintptr_t)d_in % 16 == 0) && (stride % 4 == 0);
    const uint32_t* rlen = RAG ? h->rag.d : nullptr;
    // the histogram plane has one form, in cor_kernel: with it on, tolerance mode runs the exact kernel (bit-identical plane, state
    // and reading), as a memory beyond COR_SCAN_MAX_MEMORY does
    if (h->scan && !h->hist && h->w2 >= 1.0f / COR_SCAN_MAX_MEMORY)
        cor_scan_kernel<RAG><<<(h->n_inst + CSC_WARPS - 1) / CSC_WARPS, CSC_WARPS * 32, 0, st>>> (
            d_in, stride, (int)h->n_inst, (int)nfram, aligned, h->w1, h->w2, h->d_st, h->d_res, ring, N, rboff, rlen);
    else if (h->hist)
        cor_kernel<RAG, true><<<(h->n_inst + 31) / 32, 32, 0, st>>> (d_in, stride, (int)h->n_inst, (int)nfram, aligned, h->w1, h->w2, h->d_st,
                                                                     h->d_res, ring, N, rboff, rlen, h->hist_cnt (), h->hist_sum (), h->hist_thr);
    else
        cor_kernel<RAG><<<(h->n_inst + 31) / 32, 32, 0, st>>> (d_in, stride, (int)h->n_inst, (int)nfram, aligned, h->w1, h->w2, h->d_st, h->d_res,
                                                               ring, N, rboff, rlen, nullptr, nullptr, 0.0f);
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

// A phasewheel bank with this correlation bank attached (b200m_pw_attach_cor) feeds it from its own calls, so the pair orders as
// one bank.  Each phasewheel call first enters its path on the correlation bank, as a call of the correlation bank would; a
// host-path call then runs on the correlation bank's own stream, where the correlation bank's getters look after it, and the
// phasewheel's getters follow it there.  h == nullptr (nothing attached): no-op, and the phasewheel bank's own stream.
int cor_follow (b200m_cor* h, bool host)
{
    if (!h) return 0;
    return host ? h->path.enter_host () : h->path.enter_device ();
}
cudaStream_t cor_host_stream (const b200m_cor* h, cudaStream_t pw_own) { return h ? h->path.own : pw_own; }
void cor_attach (b200m_cor* h, int d) { if (h) h->attached += d; }
}

// len: NULL (every pair runs nfram) or n_inst lengths <= nfram; they are uploaded only when they differ from the last ones
static int cor_process (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, cudaStream_t st)
{
    if (!len) return cor_launch<false> (h, d_in, stride, nfram, st, nullptr, 0, 0);
    if (h->len.empty () || memcmp (len, h->len.data (), h->n_inst * sizeof (uint32_t))) {
        if (int rc = h->rag.put (len, h->n_inst, st)) return rc;
        h->len.assign (len, len + h->n_inst);
    }
    return cor_launch<true> (h, d_in, stride, nfram, st, nullptr, 0, 0);
}

namespace b200m {
// a ragged block of the phasewheel bank this one is attached to (b200m_pw_process_ragged_*): pair i runs over its first len[i] frames,
// unfused, exactly as b200m_cor_process_ragged_* would run it
int cor_feed_ragged (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, cudaStream_t st)
{
    return cor_process (h, d_in, stride, nfram, len, st);
}
}

// b200m_cor_process_ctl_*: run[i] == 0 holds pair i, a ragged block of lengths run[i] ? nfram : 0 (NULL run: every pair runs)
static const uint32_t* cor_ctl_len (b200m_cor* h, uint32_t nfram, const uint8_t* run)
{
    if (!run) return nullptr;
    for (uint32_t i = 0; i < h->n_inst; ++i) h->ctl_len[i] = run[i] ? nfram : 0;
    return h->ctl_len.data ();
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
    h->ctl_len.assign (n_inst, 0);
    { float w[2]; b200m_design_cor (fsamp, flp, tcf, w); h->w1 = w[0]; h->w2 = w[1]; }
    cudaError_t e = cudaMalloc ((void**)&h->d_st, (size_t)5 * n_inst * sizeof (float));
    if (e == cudaSuccess) e = cudaMemset (h->d_st, 0, (size_t)5 * n_inst * sizeof (float));
    if (e == cudaSuccess) e = cudaMalloc ((void**)&h->d_res, n_inst * sizeof (float));
    if (e == cudaSuccess) e = cudaMemset (h->d_res, 0, n_inst * sizeof (float));
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags (&h->path.own, cudaStreamNonBlocking);
    if (e != cudaSuccess) { int rc = cuda_fail (e, "cor_create", __FILE__, __LINE__); b200m_cor_destroy (h); return rc; }
    *out = h;
    return 0;
}

int b200m_cor_destroy (b200m_cor* h)
{
    if (!h) return 0;
    DeviceGuard g (h->device);
    cudaDeviceSynchronize ();
    cudaFree (h->d_st); cudaFree (h->d_res); cudaFree (h->d_hist); h->rag.release (); h->path.release ();
    delete h;
    return 0;
}

// every block entry point; run: as b200m_cor_process_ctl_* (NULL: every pair runs); ragged: a b200m_cor_process_ragged_* call with
// lengths len, refused while a phasewheel bank feeds this one
static int cor_block (b200m_cor* h, const float* in, size_t stride, uint32_t nfram, const uint8_t* run, bool ragged, bool host, void* stream,
                      const uint32_t* len)
{
    return bank_call (h, in, stride, nfram, host, stream, h ? (size_t)2 * h->n_inst : 0, h ? h->n_inst : 0, len,
                      [&] {
                          if (!ragged || !h->attached) return 0;
                          return set_err (B200M_E_UNSUPPORTED, "ragged blocks: this correlation bank is attached to a phasewheel bank, whose ring advances bank-wide");
                      },
                      [&] (const float* d_in, size_t ds, cudaStream_t st, const uint32_t* rlen) {
                          return cor_process (h, d_in, ds, nfram, rlen ? rlen : cor_ctl_len (h, nfram, run), st);
                      });
}

int b200m_cor_process_ctl_device (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, const uint8_t* run, void* stream)
{
    return cor_block (h, d_in, stride, nfram, run, false, false, stream, nullptr);
}

int b200m_cor_process_device (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, void* stream)
{
    return cor_block (h, d_in, stride, nfram, nullptr, false, false, stream, nullptr);
}

int b200m_cor_process_ctl_host (b200m_cor* h, const float* in, size_t stride, uint32_t nfram, const uint8_t* run)
{
    return cor_block (h, in, stride, nfram, run, false, true, nullptr, nullptr);
}

int b200m_cor_process_host (b200m_cor* h, const float* in, size_t stride, uint32_t nfram)
{
    return cor_block (h, in, stride, nfram, nullptr, false, true, nullptr, nullptr);
}

int b200m_cor_process_ragged_device (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream)
{
    return cor_block (h, d_in, stride, nfram, nullptr, true, false, stream, len);
}

int b200m_cor_process_ragged_host (b200m_cor* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len)
{
    return cor_block (h, in, stride, nfram, nullptr, true, true, nullptr, len);
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
    cudaStream_t st = h->path.stream (stream);
    cor_clear_kernel<<<(n + 127) / 128, 128, 0, st>>> ((int)h->n_inst, i0, n, h->d_st, h->d_res);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    if (h->hist) {                                         // a cleared slot is a fresh instance for the histogram too
        B200M_CUDA (cudaMemsetAsync (h->hist_cnt () + (size_t)i0 * B200M_COR_HIST_BINS, 0,
                                     (size_t)n * B200M_COR_HIST_BINS * sizeof (unsigned long long), st));
        B200M_CUDA (cudaMemsetAsync (h->hist_sum () + i0, 0, (size_t)n * sizeof (double), st));
    }
    return 0;
}

int b200m_cor_hist_enable (b200m_cor* h, int enable, float gate_db, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    if (isnan (gate_db) || gate_db == INFINITY) return set_err (B200M_E_INVAL, "gate_db must be a number or -inf");
    DeviceGuard g (h->device);
    if (!enable) { h->hist = false; return 0; }           // the plane's memory stays for the next enable
    cudaStream_t st = h->path.stream (stream);
    if (!h->d_hist) {
        const cudaError_t e = cudaMalloc (&h->d_hist, h->hist_bytes ());
        if (e != cudaSuccess) {
            cudaGetLastError ();                               // a failed allocation is not sticky: later calls must not see it
            h->d_hist = nullptr;
            if (e == cudaErrorMemoryAllocation) return set_err (B200M_E_NOMEM, "correlation histogram of %u pairs: out of device memory", h->n_inst);
            return cuda_fail (e, "b200m_cor_hist_enable", __FILE__, __LINE__);
        }
    }
    B200M_CUDA (cudaMemsetAsync (h->d_hist, 0, h->hist_bytes (), st));
    h->hist_thr = (float)(2.0 * pow (10.0, (double)gate_db / 10.0));   // -inf dB: 0, every frame with a finite reading counts
    h->hist = true;
    return 0;
}

int b200m_cor_hist_read (b200m_cor* h, uint64_t* counts, double* sums, void* stream)
{
    if (!h || !counts || !sums) return set_err (B200M_E_INVAL, "NULL argument");
    if (!h->hist) return set_err (B200M_E_INVAL, "the correlation histogram plane is off (b200m_cor_hist_enable)");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    std::vector<unsigned char> buf (h->hist_bytes ());
    B200M_CUDA (cudaMemcpyAsync (buf.data (), h->d_hist, buf.size (), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    const size_t nc = (size_t)h->n_inst * B200M_COR_HIST_BINS * sizeof (uint64_t);
    memcpy (counts, buf.data (), nc);
    memcpy (sums, buf.data () + nc, (size_t)h->n_inst * sizeof (double));
    return 0;
}

int b200m_cor_results (b200m_cor* h, float* out, void* stream)
{
    if (!h || !out) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    B200M_CUDA (cudaMemcpyAsync (out, h->d_res, h->n_inst * sizeof (float), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_cor_state (b200m_cor* h, float* state5, void* stream)
{
    if (!h || !state5) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
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
