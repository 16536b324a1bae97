// stats.cu — the two integer-statistics meters of SURVEY.md §8(f) rank 1: bit-meter and signal-distribution histogram.
//
// bit-meter: replaces float_stats + the accumulation/window part of bim_run (src/bitmeter.c:63-105,248-327) for N
//   mono instances.  The reference walks every sample through ~70 counter increments; here one warp owns one
//   instance and processes 32 samples at a time: 23 ballots give, for every mantissa bit k, the word of lanes that
//   have it set; lanes are grouped by (effective) exponent with shuffles, and lane k adds popcounts into histogram
//   slot exp + k of a shared-memory copy of the 584-entry table — distinct lanes hit distinct slots, so there are
//   no atomics and every count is exact.
// signal-distribution histogram: replaces the sample loop of sdh_run (src/sigdistlv2.c:287-327): 361-bin histogram
//   with first-maximum tracking plus running mean / Welford variance in fp64.  The peak tracking and the Welford
//   recurrence (one fp64 division per sample) are order dependent, so one lane owns one instance and walks its block
//   serially from a [32 x 64] cp.async tile; the 361 bins of 32 instances live in shared memory ([bin][lane]).
// Integer results are bit-exact by construction; the fp64 statistics use the reference's operation order.
#include <math.h>
#include <stdlib.h>
#include "common.cuh"

namespace b200m {

constexpr int BIM_LEN = 584;                                // BIM_LAST, src/uris.h:52-60
constexpr int BIM_WARPS = 4;

// state per instance: hist[584], cnt[8] = zero pos nan inf den, minmax[2], st[4] = integrating average resync closed, itime;
// the snapshot published when the ~5 fps window closes: pub_hist[584], pub_cnt[8], pub_mm[2], pub_itime.
// One run of bim_run (src/bitmeter.c:248-327) per instance: acquisition (skipped while paused or at the 2^31 cap), then the
// window clock; a closing window publishes the warp's shared-memory histogram and, in windowed mode, clears the statistics.
// RAG (b200m_bim_run_ragged_*): instance inst runs bim_run over its first rlen[inst] frames, with the window limit of that run
// length, fps_tab[rlen[inst]] (:264, the host's fps_limit of every block length); rlen 0: not run, only its closed flag reads 0.
// The run length then sits in a register, not in the parameter bank: 12 CTAs per SM (40 registers) instead of 16 keep it unspilled.
template <bool RAG>
__global__ void __launch_bounds__ (BIM_WARPS * 32, RAG ? 12 : 16)
bim_kernel (const float* __restrict__ in, size_t stride, int n_inst, int nfram, int fps_limit, int32_t* __restrict__ hist,
            int32_t* __restrict__ cnt, float* __restrict__ minmax, int32_t* __restrict__ st, int64_t* __restrict__ itime,
            int32_t* __restrict__ pub_hist, int32_t* __restrict__ pub_cnt, float* __restrict__ pub_mm, int64_t* __restrict__ pub_itime,
            const uint32_t* __restrict__ rlen, const int32_t* __restrict__ fps_tab)
{
    __shared__ int32_t sh[BIM_WARPS][BIM_LEN];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int inst = blockIdx.x * BIM_WARPS + w;
    if (inst >= n_inst) return;
    if (RAG) {                                               // one warp per instance: the length is warp-uniform
        nfram = (int)rlen[inst];
        if (nfram == 0) { if (lane == 0) st[4 * inst + 3] = 0; return; }
        fps_limit = fps_tab[nfram];
    }
    const int integrating = st[4 * inst], average = st[4 * inst + 1];
    int64_t it = itime[inst];
    bool acc = false;
    if (integrating && it < 2147483647) {                    // :248-262
        if (it > 2147483647 - nfram) it = 2147483647;
        else { acc = true; it += nfram; }
    }
    int resync = st[4 * inst + 2] + nfram;                   // :264-267
    bool closed = resync >= fps_limit;
    if (closed) resync = resync % fps_limit;
    // every lane computed the same flags; as warp votes the compiler knows them to be uniform, so the ballots below need no
    // divergent-path code
    acc = __all_sync (0xffffffffu, acc); closed = __all_sync (0xffffffffu, closed);
    int32_t* h = sh[w];
    int32_t* c = cnt + (size_t)inst * 8;
    const size_t base = (size_t)inst * BIM_LEN;
    if (acc || closed) {
        for (int i = lane; i < BIM_LEN; i += 32) h[i] = hist[base + i];
        int c_zero = 0, c_pos = 0, c_nan = 0, c_inf = 0, c_den = 0;
        float mn = minmax[2 * inst], mx = minmax[2 * inst + 1];
        const float* row = in + (size_t)inst * stride;
        __syncwarp ();
        for (int j0 = 0; acc && j0 < nfram; j0 += 32) {
            const bool have = (j0 + lane) < nfram;
            const float f = have ? row[j0 + lane] : 0.0f;
            const uint32_t v = __float_as_uint (f);
            const uint32_t e = (v >> 23) & 255u, mant = v & 0x7fffffu;
            const bool is_special = have && e == 255;            // :70-76
            const bool is_zero = have && e == 0 && mant == 0;    // :77-79
            const bool counted = have && !is_special && !is_zero;
            const bool normal = counted && e > 0;
            c_inf += __popc (__ballot_sync (0xffffffffu, is_special && mant == 0));
            c_nan += __popc (__ballot_sync (0xffffffffu, is_special && mant != 0));
            c_zero += __popc (__ballot_sync (0xffffffffu, is_zero));
            c_den += __popc (__ballot_sync (0xffffffffu, counted && e == 0));
            c_pos += __popc (__ballot_sync (0xffffffffu, counted && !(v >> 31)));
            const unsigned valid = __ballot_sync (0xffffffffu, counted);
            const unsigned nmask = __ballot_sync (0xffffffffu, normal);
            // min / max of |sample| over normal numbers (:88-91)
            float a = normal ? fabsf (f) : 0.0f, bmin = normal ? fabsf (f) : INFINITY;
#pragma unroll
            for (int o = 16; o; o >>= 1) { a = fmaxf (a, __shfl_xor_sync (0xffffffffu, a, o)); bmin = fminf (bmin, __shfl_xor_sync (0xffffffffu, bmin, o)); }
            if (a > mx) mx = a;
            if (bmin < mn) mn = bmin;
            // lane k keeps the word of lanes whose mantissa bit k is set
            unsigned myw = 0;
#pragma unroll
            for (int k = 0; k < 23; ++k) { const unsigned wk = __ballot_sync (0xffffffffu, counted && (mant >> k & 1u)); if (lane == k) myw = wk; }
            if (lane < 23) h[560 + lane] += __popc (myw & valid);                          // BIM_DSET + k
            const uint32_t ee = e ? e : 1u;                      // "E-126 not E-127 for denormals" (:95)
            unsigned rem = valid;
            while (rem) {
                const int leader = __ffs (rem) - 1;
                const uint32_t ge = __shfl_sync (0xffffffffu, ee, leader);
                const unsigned grp = __ballot_sync (0xffffffffu, counted && ee == ge);
                rem &= ~grp;
                if (lane < 23) {
                    h[0 + ge + lane] += __popc (grp);                                      // BIM_DHIT + exp + k
                    h[280 + ge + lane] += __popc (grp & myw);                              // BIM_DONE + exp + k
                } else if (lane == 23) {
                    const int nn = __popc (grp & nmask);
                    h[23 + ge] += nn;                                                      // BIM_NHIT + exp
                    h[303 + ge] += nn;                                                     // BIM_NONE + exp
                }
                __syncwarp ();
            }
        }
        __syncwarp ();
        const int32_t t0 = c[0] + c_zero, t1 = c[1] + c_pos, t2 = c[2] + c_nan, t3 = c[3] + c_inf, t4 = c[4] + c_den;
        __syncwarp ();                                       // every lane has read c before lane 0 rewrites it
        if (closed) {                                        // publish (:267-291); windowed mode then bim_clear (:46-54,323-325)
            for (int i = lane; i < BIM_LEN; i += 32) { pub_hist[base + i] = h[i]; hist[base + i] = average ? h[i] : 0; }
            if (lane == 0) {
                int32_t* pc = pub_cnt + (size_t)inst * 8;
                pc[0] = t0; pc[1] = t1; pc[2] = t2; pc[3] = t3; pc[4] = t4;
                pub_mm[2 * inst] = mn; pub_mm[2 * inst + 1] = mx; pub_itime[inst] = it;
                if (!average) { mn = INFINITY; mx = 0.0f; it = 0; }
                c[0] = average ? t0 : 0; c[1] = average ? t1 : 0; c[2] = t2; c[3] = t3; c[4] = t4;
                minmax[2 * inst] = mn; minmax[2 * inst + 1] = mx;
            }
        } else {
            for (int i = lane; i < BIM_LEN; i += 32) hist[base + i] = h[i];
            if (lane == 0) { c[0] = t0; c[1] = t1; c[2] = t2; c[3] = t3; c[4] = t4; minmax[2 * inst] = mn; minmax[2 * inst + 1] = mx; }
        }
    }
    if (lane == 0) { itime[inst] = it; st[4 * inst + 2] = resync; st[4 * inst + 3] = closed; }
}

// B200M_CTL_* on instances [i0, i0 + n_sel) (:207-231): START / PAUSE / AVERAGE / WINDOWED set a flag; RESET is bim_reset
// (:56-59: statistics, all counters, integration time); CLEAR also restores what bim_instantiate sets (:146-158): integrating,
// windowed, the window clock at 0, and an empty published snapshot
__global__ void bim_control_kernel (int i0, int n_sel, int cmd, int32_t* hist, int32_t* cnt, float* minmax, int32_t* st, int64_t* itime,
                                    int32_t* pub_hist, int32_t* pub_cnt, float* pub_mm, int64_t* pub_itime)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool clear = cmd == B200M_CTL_CLEAR, reset = clear || cmd == B200M_CTL_RESET;
    if (reset && i < (size_t)n_sel * BIM_LEN) {
        hist[(size_t)i0 * BIM_LEN + i] = 0;
        if (clear) pub_hist[(size_t)i0 * BIM_LEN + i] = 0;
    }
    if (i >= (size_t)n_sel) return;
    const size_t k = i0 + i;
    int32_t* s = st + 4 * k;
    switch (cmd) {
    case B200M_CTL_START: s[0] = 1; break;
    case B200M_CTL_PAUSE: s[0] = 0; break;
    case B200M_CTL_AVERAGE: s[1] = 1; break;
    case B200M_CTL_WINDOWED: s[1] = 0; break;
    default:
        if (clear) {
            s[0] = 1; s[1] = 0; s[2] = 0; s[3] = 0;
            for (int j = 0; j < 8; ++j) pub_cnt[8 * k + j] = 0;
            pub_mm[2 * k] = 0.0f; pub_mm[2 * k + 1] = 0.0f; pub_itime[k] = 0;
        }
        minmax[2 * k] = INFINITY; minmax[2 * k + 1] = 0.0f;
        for (int j = 0; j < 5; ++j) cnt[8 * k + j] = 0;
        itime[k] = 0;
        break;
    }
}

// ---------------------------------------------------------------------------------------------------------------
constexpr int SDH_BINS = 361, SDH_T = 64, SDH_P = SDH_T + 4, SDH_STAGES = 2;
constexpr int SDH_BP = 33;                                  // bin pitch: [bin][lane] padded -> conflict-free both ways
constexpr int SDH_SMEM = (SDH_BINS * SDH_BP + 3 + SDH_STAGES * 32 * SDH_P) * 4;   // ~65 KB per (one-warp) CTA

// per instance: hist[361] (layout [n][361]), ip[2] = max count, peak bin; dp[3] = avg, var_m, var_s; integrating, itime.
// A lane whose instance is paused or at the 2^31-sample cap (src/sigdistlv2.c:287) scans nothing; a CTA with no such lane exits.
// RAG (b200m_sdh_run_ragged_*): lane's instance runs sdh_run over its first rlen[inst] frames (0: not run); the warp stages tiles
// up to its longest running length.
template <bool RAG>
__global__ void __launch_bounds__ (32)
sdh_kernel (const float* __restrict__ in, size_t stride, int n_inst, int nfram, int aligned, const int32_t* __restrict__ integrating,
            int64_t* __restrict__ itime, int32_t* __restrict__ hist, int32_t* __restrict__ ip, double* __restrict__ dp,
            const uint32_t* __restrict__ rlen)
{
    extern __shared__ __align__ (16) int32_t sdh_smem[];
    int32_t* sb = sdh_smem;                                  // [361][33]
    float* tile = reinterpret_cast<float*> (sdh_smem + ((SDH_BINS * SDH_BP + 3) & ~3));
    const int lane = threadIdx.x, i0 = blockIdx.x * 32;
    const int inst = min (i0 + lane, n_inst - 1);
    const bool live = (i0 + lane) < n_inst;
    const int rl = RAG ? (live ? (int)rlen[inst] : 0) : nfram;                 // this instance's run length
    int64_t it = itime[inst];
    bool run = live && (!RAG || rl > 0) && integrating[inst] && it < 2147483647;
    if (run && it > 2147483647 - rl) { it = 2147483647; run = false; }
    if (!__any_sync (0xffffffffu, run)) { if (live) itime[inst] = it; return; }
    const int wend = RAG ? __reduce_max_sync (0xffffffffu, run ? rl : 0) : nfram;   // frames the warp stages
    const double itime0 = (double)it;
    const int ntiles = (wend + SDH_T - 1) / SDH_T;
    auto issue = [&] (int t) {
        if (t < ntiles) {
            float* dst = tile + (t % SDH_STAGES) * (32 * SDH_P);
            const int s0 = t * SDH_T;
            if (aligned) {
                const int c4 = (lane & 15) * 4;
                const int left = (wend - (s0 + c4)) * 4;
                const int nb = left >= 16 ? 16 : (left > 0 ? left : 0);
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const int r = 2 * i + (lane >> 4);
                    const int ir = min (i0 + r, n_inst - 1);
                    cp_async16 (dst + r * SDH_P + c4, nb ? in + (size_t)ir * stride + s0 + c4 : in, nb);
                }
            } else {
                for (int r = 0; r < 32; ++r) {
                    const int ir = min (i0 + r, n_inst - 1);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const int c = lane + 32 * hh; const bool ok = (s0 + c) < wend;
                        cp_async4 (dst + r * SDH_P + c, ok ? in + (size_t)ir * stride + s0 + c : in, ok ? 4 : 0);
                    }
                }
            }
        }
        cp_async_commit ();
    };
    issue (0);
    // histogram rows -> smem, transposed so that lane = instance is conflict free
    for (int r = 0; r < 32; ++r) {
        const int ir = min (i0 + r, n_inst - 1);
        for (int b = lane; b < SDH_BINS; b += 32) sb[b * SDH_BP + r] = hist[(size_t)ir * SDH_BINS + b];
    }
    int peak_cnt = ip[2 * inst], peak_bin = ip[2 * inst + 1];
    double avg = dp[3 * inst], vm = dp[3 * inst + 1], vs = dp[3 * inst + 2];
    __syncwarp ();
    for (int t = 0; t < ntiles; ++t) {
        issue (t + 1);
        cp_async_wait<1> ();
        __syncwarp ();
        const float* row = tile + (t % SDH_STAGES) * (32 * SDH_P) + lane * SDH_P;
        const int len = run ? min (SDH_T, rl - t * SDH_T) : 0;
        for (int j = 0; j < len; ++j) {                      // src/sigdistlv2.c:303-318
            const float val = row[j];
            const float r = rintf (__fadd_rn (180.f, __fmul_rn (val, 150.f)));
            if (!(r >= 0.f && r < 361.f)) continue;          // (int) of NaN / out of range is INT_MIN on x86: "bin < 0"
            const int bin = (int)r;
            const int nc = ++sb[bin * SDH_BP + lane];
            if (nc > peak_cnt) { peak_cnt = nc; peak_bin = bin; }
            avg = __dadd_rn (avg, (double)val);
            const double m1 = vm, cnt = __dadd_rn (itime0, (double)(t * SDH_T + j + 1));
            vm = __dadd_rn (vm, __ddiv_rn (__dsub_rn ((double)val, vm), cnt));
            vs = __dadd_rn (vs, __dmul_rn (__dsub_rn ((double)val, vm), __dsub_rn ((double)val, m1)));
        }
        __syncwarp ();
    }
    cp_async_wait<0> ();
    __syncwarp ();
    for (int r = 0; r < 32; ++r) {
        if (i0 + r >= n_inst) break;
        for (int b = lane; b < SDH_BINS; b += 32) hist[(size_t)(i0 + r) * SDH_BINS + b] = sb[b * SDH_BP + r];
    }
    if (run) { ip[2 * inst] = peak_cnt; ip[2 * inst + 1] = peak_bin; dp[3 * inst] = avg; dp[3 * inst + 1] = vm; dp[3 * inst + 2] = vs; it += rl; }
    if (live) itime[inst] = it;
}

// B200M_CTL_* on instances [i0, i0 + n_sel): START / PAUSE (sdh_integrate, :233-241); RESET = sdh_reset (:141-150);
// CLEAR = sdh_reset with integration off, i.e. sdh_instantiate
__global__ void sdh_control_kernel (int i0, int n_sel, int cmd, int32_t* integrating, int64_t* itime, int32_t* hist, int32_t* ip, double* dp)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool reset = cmd == B200M_CTL_RESET || cmd == B200M_CTL_CLEAR;
    if (reset && i < (size_t)n_sel * SDH_BINS) hist[(size_t)i0 * SDH_BINS + i] = 0;
    if (i >= (size_t)n_sel) return;
    const size_t k = i0 + i;
    if (cmd == B200M_CTL_START || cmd == B200M_CTL_PAUSE || cmd == B200M_CTL_CLEAR) integrating[k] = cmd == B200M_CTL_START;
    if (reset) { ip[2 * k] = 0; ip[2 * k + 1] = -1; dp[3 * k] = 0; dp[3 * k + 1] = 0; dp[3 * k + 2] = 0; itime[k] = 0; }
}

}  // namespace b200m

using namespace b200m;

struct b200m_bim {
    int device; uint32_t n_inst; double rate;
    int32_t *d_hist = nullptr, *d_cnt = nullptr, *d_st = nullptr; float* d_mm = nullptr; int64_t* d_itime = nullptr;
    // the statistics as they stood when an instance's last ~5 fps window closed, i.e. what bim_run publishes before bim_clear (:267-326)
    int32_t *d_pub_hist = nullptr, *d_pub_cnt = nullptr; float* d_pub_mm = nullptr; int64_t* d_pub_itime = nullptr;
    int resync = 0; bool window_closed = false;                // the window clock of a bank driven only bank-wide (b200m_bim_window_closed)
    RaggedLen rag;                                             // the lengths of a ragged block
    int32_t* d_fps = nullptr;                                  // fps_limit of every block length 0 .. B200M_MAX_BLOCK (ragged blocks)
    BankPath path;
};
struct b200m_sdh {
    int device; uint32_t n_inst; double rate;
    int32_t *d_hist = nullptr, *d_ip = nullptr, *d_integ = nullptr; double* d_dp = nullptr; int64_t* d_itime = nullptr;
    RaggedLen rag;
    BankPath path;
};

static int bim_control (b200m_bim* h, int32_t inst, int cmd, cudaStream_t st)
{
    if (cmd < B200M_CTL_START || cmd > B200M_CTL_CLEAR) return set_err (B200M_E_INVAL, "unknown control %d", cmd);
    if (inst < -1 || inst >= (int64_t)h->n_inst) return set_err (B200M_E_INVAL, "bad instance %d", inst);
    const uint32_t i0 = inst < 0 ? 0 : (uint32_t)inst, n = inst < 0 ? h->n_inst : 1;
    const size_t threads = cmd == B200M_CTL_RESET || cmd == B200M_CTL_CLEAR ? (size_t)n * BIM_LEN : n;
    bim_control_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>> ((int)i0, (int)n, cmd, h->d_hist, h->d_cnt, h->d_mm, h->d_st, h->d_itime,
                                                                            h->d_pub_hist, h->d_pub_cnt, h->d_pub_mm, h->d_pub_itime);
    B200M_LAUNCHED (1);
    if (inst < 0 && cmd == B200M_CTL_CLEAR) { h->resync = 0; h->window_closed = false; }
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

// rlen: NULL, or the host array of n_inst lengths of a ragged block (bank_call passes it only when some length differs from n)
// the ~5 fps window limit of a block of n frames (:264)
static int bim_fps_limit (double rate, uint32_t n) { return n * ceil (rate / (5.f * n)); }

static int bim_run (b200m_bim* h, const float* d_in, size_t stride, uint32_t n, const uint32_t* rlen, cudaStream_t st)
{
    // bim_run (:248-327) for every instance: acquisition, the ~5 fps window clock, publish + windowed-mode clear
    const int fps_limit = bim_fps_limit (h->rate, n);
    const unsigned grid = (h->n_inst + BIM_WARPS - 1) / BIM_WARPS;
    if (rlen) {
        // each instance's window limit follows its own run length; the bank-wide clock stands still and reads "not closed"
        if (int rc = h->rag.put (rlen, h->n_inst, st)) return rc;
        bim_kernel<true><<<grid, BIM_WARPS * 32, 0, st>>> (d_in, stride, (int)h->n_inst, (int)n, fps_limit, h->d_hist, h->d_cnt, h->d_mm, h->d_st,
                                                           h->d_itime, h->d_pub_hist, h->d_pub_cnt, h->d_pub_mm, h->d_pub_itime, h->rag.d, h->d_fps);
        B200M_LAUNCHED (1);
        h->window_closed = false;
        B200M_CUDA (cudaGetLastError ());
        return 0;
    }
    bim_kernel<false><<<grid, BIM_WARPS * 32, 0, st>>> (d_in, stride, (int)h->n_inst, (int)n, fps_limit, h->d_hist, h->d_cnt, h->d_mm,
                                                        h->d_st, h->d_itime, h->d_pub_hist, h->d_pub_cnt, h->d_pub_mm, h->d_pub_itime, nullptr, nullptr);
    B200M_LAUNCHED (1);
    h->resync += n;
    h->window_closed = h->resync >= fps_limit;
    if (h->window_closed) h->resync = h->resync % fps_limit;
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

static int sdh_control (b200m_sdh* h, int32_t inst, int cmd, cudaStream_t st)
{
    if (cmd != B200M_CTL_START && cmd != B200M_CTL_PAUSE && cmd != B200M_CTL_RESET && cmd != B200M_CTL_CLEAR)
        return set_err (B200M_E_INVAL, "unknown control %d", cmd);
    if (inst < -1 || inst >= (int64_t)h->n_inst) return set_err (B200M_E_INVAL, "bad instance %d", inst);
    const uint32_t i0 = inst < 0 ? 0 : (uint32_t)inst, n = inst < 0 ? h->n_inst : 1;
    const size_t threads = cmd == B200M_CTL_RESET || cmd == B200M_CTL_CLEAR ? (size_t)n * SDH_BINS : n;
    sdh_control_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>> ((int)i0, (int)n, cmd, h->d_integ, h->d_itime, h->d_hist, h->d_ip, h->d_dp);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

static int sdh_run (b200m_sdh* h, const float* d_in, size_t stride, uint32_t n, const uint32_t* rlen, cudaStream_t st)
{
    const int aligned = ((uintptr_t)d_in % 16 == 0) && (stride % 4 == 0);
    const unsigned grid = (h->n_inst + 31) / 32;
    if (rlen) {
        if (int rc = h->rag.put (rlen, h->n_inst, st)) return rc;
        sdh_kernel<true><<<grid, 32, SDH_SMEM, st>>> (d_in, stride, (int)h->n_inst, (int)n, aligned, h->d_integ, h->d_itime, h->d_hist, h->d_ip, h->d_dp,
                                                      h->rag.d);
    } else {
        sdh_kernel<false><<<grid, 32, SDH_SMEM, st>>> (d_in, stride, (int)h->n_inst, (int)n, aligned, h->d_integ, h->d_itime, h->d_hist, h->d_ip, h->d_dp,
                                                       nullptr);
    }
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

extern "C" {

// ---- bit-meter ---------------------------------------------------------------------------------------------
int b200m_bim_create (b200m_bim** out, int device, uint32_t n_inst, double rate)
{
    if (!out) return set_err (B200M_E_INVAL, "NULL out pointer");
    *out = nullptr;
    if (n_inst == 0 || !(rate >= 1000.0)) return set_err (B200M_E_INVAL, "bad n_inst/rate");
    if (b200m_device_count () <= 0) return set_err (B200M_E_NODEVICE, "no CUDA device: b200meters has no CPU path");
    DeviceGuard g (device);
    if (!g.ok) return set_err (B200M_E_NODEVICE, "cannot select CUDA device %d", device);
    b200m_bim* h = new (std::nothrow) b200m_bim;
    if (!h) return set_err (B200M_E_NOMEM, "host allocation failed");
    h->device = device; h->n_inst = n_inst; h->rate = rate;
    cudaError_t e = cudaSuccess;
    auto A = [&] (void** p, size_t bytes) { if (e == cudaSuccess) { e = cudaMalloc (p, bytes); if (e == cudaSuccess) e = cudaMemset (*p, 0, bytes); } };
    A ((void**)&h->d_hist, (size_t)n_inst * BIM_LEN * 4); A ((void**)&h->d_cnt, (size_t)n_inst * 8 * 4); A ((void**)&h->d_mm, (size_t)n_inst * 2 * 4);
    A ((void**)&h->d_st, (size_t)n_inst * 4 * 4); A ((void**)&h->d_itime, (size_t)n_inst * 8);
    A ((void**)&h->d_pub_hist, (size_t)n_inst * BIM_LEN * 4); A ((void**)&h->d_pub_cnt, (size_t)n_inst * 8 * 4); A ((void**)&h->d_pub_mm, (size_t)n_inst * 2 * 4);
    A ((void**)&h->d_pub_itime, (size_t)n_inst * 8); A ((void**)&h->d_fps, (B200M_MAX_BLOCK + 1) * 4);
    if (e == cudaSuccess) {
        static_assert (B200M_MAX_BLOCK <= 8192, "fps table on the stack");
        int32_t fps[B200M_MAX_BLOCK + 1] = {0};
        for (uint32_t n = 1; n <= B200M_MAX_BLOCK; ++n) fps[n] = bim_fps_limit (rate, n);
        e = cudaMemcpy (h->d_fps, fps, sizeof (fps), cudaMemcpyHostToDevice);
    }
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags (&h->path.own, cudaStreamNonBlocking);
    if (e == cudaSuccess) { bim_control (h, -1, B200M_CTL_CLEAR, nullptr); e = cudaDeviceSynchronize (); }      // bim_instantiate (:146-158)
    if (e != cudaSuccess) { int rc = cuda_fail (e, "bim_create", __FILE__, __LINE__); b200m_bim_destroy (h); return rc; }
    *out = h;
    return 0;
}
int b200m_bim_destroy (b200m_bim* h)
{
    if (!h) return 0;
    DeviceGuard g (h->device);
    cudaDeviceSynchronize ();
    cudaFree (h->d_hist); cudaFree (h->d_cnt); cudaFree (h->d_mm); cudaFree (h->d_st); cudaFree (h->d_itime);
    cudaFree (h->d_pub_hist); cudaFree (h->d_pub_cnt); cudaFree (h->d_pub_mm); cudaFree (h->d_pub_itime); cudaFree (h->d_fps); h->rag.release ();
    h->path.release ();
    delete h;
    return 0;
}
int b200m_bim_control (b200m_bim* h, int cmd, void* stream) { return b200m_bim_control_inst (h, -1, cmd, stream); }
int b200m_bim_control_inst (b200m_bim* h, int32_t inst, int cmd, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    DeviceGuard g (h->device);
    return bim_control (h, inst, cmd, h->path.stream (stream));   // CTL_* handling of bim_run (:207-231)
}
static int bim_block (b200m_bim* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len, bool host, void* stream)
{
    return bank_call (h, in, stride, nfram, host, stream, h ? h->n_inst : 0, h ? h->n_inst : 0, len, no_check,
                      [&] (const float* d_in, size_t ds, cudaStream_t st, const uint32_t* rlen) { return bim_run (h, d_in, ds, nfram, rlen, st); });
}
int b200m_bim_run_device (b200m_bim* h, const float* d_in, size_t stride, uint32_t nfram, void* stream) { return bim_block (h, d_in, stride, nfram, nullptr, false, stream); }
int b200m_bim_run_host (b200m_bim* h, const float* in, size_t stride, uint32_t nfram) { return bim_block (h, in, stride, nfram, nullptr, true, nullptr); }
int b200m_bim_run_ragged_device (b200m_bim* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream)
{
    return bim_block (h, d_in, stride, nfram, len, false, stream);
}
int b200m_bim_run_ragged_host (b200m_bim* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len)
{
    return bim_block (h, in, stride, nfram, len, true, nullptr);
}
// one row of statistics (hist, counters, min/max, integration time), live or published, of instances [i0, i0 + n)
static int bim_copy_rows (b200m_bim* h, bool pub, uint32_t i0, uint32_t n, int32_t* hist, int32_t* cnt5, float* mm2, int64_t* itime, cudaStream_t st)
{
    const int32_t* dh = pub ? h->d_pub_hist : h->d_hist; const int32_t* dc = pub ? h->d_pub_cnt : h->d_cnt;
    const float* dm = pub ? h->d_pub_mm : h->d_mm; const int64_t* di = pub ? h->d_pub_itime : h->d_itime;
    if (hist) B200M_CUDA (cudaMemcpyAsync (hist, dh + (size_t)i0 * BIM_LEN, (size_t)n * BIM_LEN * 4, cudaMemcpyDeviceToHost, st));
    if (cnt5) B200M_CUDA (cudaMemcpy2DAsync (cnt5, 5 * 4, dc + (size_t)i0 * 8, 8 * 4, 5 * 4, n, cudaMemcpyDeviceToHost, st));
    if (mm2) B200M_CUDA (cudaMemcpyAsync (mm2, dm + (size_t)i0 * 2, (size_t)n * 2 * 4, cudaMemcpyDeviceToHost, st));
    if (itime) B200M_CUDA (cudaMemcpyAsync (itime, di + i0, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    return 0;
}
int b200m_bim_results (b200m_bim* h, uint32_t inst, int32_t* hist584, int32_t* cnt5, float* minmax2, int64_t* integration_time, void* stream)
{
    if (!h || inst >= h->n_inst) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    if (int rc = bim_copy_rows (h, false, inst, 1, hist584, cnt5, minmax2, integration_time, st)) return rc;
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}
int b200m_bim_window_closed (const b200m_bim* h) { return h && h->window_closed ? 1 : 0; }
int b200m_bim_published (b200m_bim* h, uint32_t inst, int32_t* hist584, int32_t* cnt5, float* minmax2, int64_t* integration_time, void* stream)
{
    if (!h || inst >= h->n_inst) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    if (int rc = bim_copy_rows (h, true, inst, 1, hist584, cnt5, minmax2, integration_time, st)) return rc;
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}
int b200m_bim_results_all (b200m_bim* h, int32_t* hist, int32_t* cnt5, float* minmax2, int64_t* integration_time, int32_t* closed,
                           int32_t* pub_hist, int32_t* pub_cnt5, float* pub_minmax2, int64_t* pub_integration_time, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    if (int rc = bim_copy_rows (h, false, 0, h->n_inst, hist, cnt5, minmax2, integration_time, st)) return rc;
    if (int rc = bim_copy_rows (h, true, 0, h->n_inst, pub_hist, pub_cnt5, pub_minmax2, pub_integration_time, st)) return rc;
    if (closed) B200M_CUDA (cudaMemcpy2DAsync (closed, 4, h->d_st + 3, 4 * 4, 4, h->n_inst, cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

// ---- signal distribution histogram -------------------------------------------------------------------------
int b200m_sdh_create (b200m_sdh** out, int device, uint32_t n_inst, double rate)
{
    if (!out) return set_err (B200M_E_INVAL, "NULL out pointer");
    *out = nullptr;
    if (n_inst == 0 || !(rate >= 1000.0)) return set_err (B200M_E_INVAL, "bad n_inst/rate");
    if (b200m_device_count () <= 0) return set_err (B200M_E_NODEVICE, "no CUDA device: b200meters has no CPU path");
    DeviceGuard g (device);
    if (!g.ok) return set_err (B200M_E_NODEVICE, "cannot select CUDA device %d", device);
    b200m_sdh* h = new (std::nothrow) b200m_sdh;
    if (!h) return set_err (B200M_E_NOMEM, "host allocation failed");
    h->device = device; h->n_inst = n_inst; h->rate = rate;
    cudaError_t e = cudaSuccess;
    auto A = [&] (void** p, size_t bytes) { if (e == cudaSuccess) { e = cudaMalloc (p, bytes); if (e == cudaSuccess) e = cudaMemset (*p, 0, bytes); } };
    A ((void**)&h->d_hist, (size_t)n_inst * SDH_BINS * 4); A ((void**)&h->d_ip, (size_t)n_inst * 2 * 4); A ((void**)&h->d_dp, (size_t)n_inst * 3 * 8);
    A ((void**)&h->d_integ, (size_t)n_inst * 4); A ((void**)&h->d_itime, (size_t)n_inst * 8);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags (&h->path.own, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaFuncSetAttribute (sdh_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SDH_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute (sdh_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SDH_SMEM);
    if (e == cudaSuccess) { sdh_control (h, -1, B200M_CTL_CLEAR, nullptr); e = cudaDeviceSynchronize (); }        // sdh_instantiate (:141-150)
    if (e != cudaSuccess) { int rc = cuda_fail (e, "sdh_create", __FILE__, __LINE__); b200m_sdh_destroy (h); return rc; }
    *out = h;
    return 0;
}
int b200m_sdh_destroy (b200m_sdh* h)
{
    if (!h) return 0;
    DeviceGuard g (h->device);
    cudaDeviceSynchronize ();
    cudaFree (h->d_hist); cudaFree (h->d_ip); cudaFree (h->d_dp); cudaFree (h->d_integ); cudaFree (h->d_itime); h->rag.release (); h->path.release ();
    delete h;
    return 0;
}
int b200m_sdh_control (b200m_sdh* h, int cmd, void* stream) { return b200m_sdh_control_inst (h, -1, cmd, stream); }
int b200m_sdh_control_inst (b200m_sdh* h, int32_t inst, int cmd, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    DeviceGuard g (h->device);
    return sdh_control (h, inst, cmd, h->path.stream (stream));   // sdh_integrate / sdh_reset (:233-241)
}
static int sdh_block (b200m_sdh* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len, bool host, void* stream)
{
    return bank_call (h, in, stride, nfram, host, stream, h ? h->n_inst : 0, h ? h->n_inst : 0, len, no_check,
                      [&] (const float* d_in, size_t ds, cudaStream_t st, const uint32_t* rlen) { return sdh_run (h, d_in, ds, nfram, rlen, st); });
}
int b200m_sdh_run_device (b200m_sdh* h, const float* d_in, size_t stride, uint32_t nfram, void* stream) { return sdh_block (h, d_in, stride, nfram, nullptr, false, stream); }
int b200m_sdh_run_host (b200m_sdh* h, const float* in, size_t stride, uint32_t nfram) { return sdh_block (h, in, stride, nfram, nullptr, true, nullptr); }
int b200m_sdh_run_ragged_device (b200m_sdh* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream)
{
    return sdh_block (h, d_in, stride, nfram, len, false, stream);
}
int b200m_sdh_run_ragged_host (b200m_sdh* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len)
{
    return sdh_block (h, in, stride, nfram, len, true, nullptr);
}
static int sdh_copy_rows (b200m_sdh* h, uint32_t i0, uint32_t n, int32_t* hist, int32_t* mp2, double* atv3, int64_t* itime, cudaStream_t st)
{
    if (hist) B200M_CUDA (cudaMemcpyAsync (hist, h->d_hist + (size_t)i0 * SDH_BINS, (size_t)n * SDH_BINS * 4, cudaMemcpyDeviceToHost, st));
    if (mp2) B200M_CUDA (cudaMemcpyAsync (mp2, h->d_ip + (size_t)i0 * 2, (size_t)n * 2 * 4, cudaMemcpyDeviceToHost, st));
    if (atv3) B200M_CUDA (cudaMemcpyAsync (atv3, h->d_dp + (size_t)i0 * 3, (size_t)n * 3 * 8, cudaMemcpyDeviceToHost, st));
    if (itime) B200M_CUDA (cudaMemcpyAsync (itime, h->d_itime + i0, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    return 0;
}
int b200m_sdh_results (b200m_sdh* h, uint32_t inst, int32_t* hist361, int32_t* max_peak2, double* avg_tmp_var3, int64_t* integration_time, void* stream)
{
    if (!h || inst >= h->n_inst) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    if (int rc = sdh_copy_rows (h, inst, 1, hist361, max_peak2, avg_tmp_var3, integration_time, st)) return rc;
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}
int b200m_sdh_results_all (b200m_sdh* h, int32_t* hist, int32_t* max_peak2, double* avg_tmp_var3, int64_t* integration_time, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    if (int rc = sdh_copy_rows (h, 0, h->n_inst, hist, max_peak2, avg_tmp_var3, integration_time, st)) return rc;
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

}  // extern "C"
