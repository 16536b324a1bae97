// dr14.cu — DR-14 / TPnRMS bank: dr14_run (src/dr14.c:354-482) for N mono or stereo instances at once.
//
// Per run() the reference does, per channel: Kmeterdsp::process + TruePeakdsp::process (the C3 kernels of tpk.cu), in
// DR mode the 3 s-window sums rms_sum += v*v, peak_cur = MAX (peak_cur, v) with dr14_calc_rms_score at each window end
// (:285-352: silence gate, 8000-bin RMS histogram in 0.01 dB steps, mean of the loudest 20 % of the windows, second
// highest window peak), then read() of both meters and the port arithmetic (:418-462).
//
// Mapping: the window sums ride on the process() kernel as an extra lane role (TpkDr, tpk_internal.cuh) so the
// input is still read once.  The bank keeps one sample clock on the host; each instance's window phase (the bank time of
// its last reset_peaks, mod the window length) is device state written only by the control kernel, and each DR lane
// derives its instance's window end in the block from it.  The host mirrors the phases (an ordered count of the distinct
// ones), so the scoring kernel is launched only in blocks where some window closes.  The scoring is one warp per instance:
// the top-down histogram walk is a ballot over 32 bins at a time, accumulated in exactly the reference's bin order.  Port
// values are computed on the device with the glibc-exact log10f (common.cuh), so every float equals the reference's.
#include <math.h>
#include <stdlib.h>
#include <map>
#include <vector>
#include "common.cuh"
#include "tpk_internal.cuh"

namespace b200m {

constexpr int DR_HISTBINS = 8000;           // -80 dB .. 0 dB in 0.01 dB steps (src/dr14.c:45)

B200M_DEV float dr_coeff_to_db (const float coeff)            // coeff_to_db (:236-239)
{
    if ((double)coeff < .0001) return -80.0f;
    return __fmul_rn (20.0f, log10f_glibc (coeff));
}

// (int) of a float as the reference's x86 build converts it (cvttss2si: NaN / out of range -> INT_MIN)
B200M_DEV int dr_f2i (const float f)
{
    if (!(f >= -2147483648.0f && f < 2147483648.0f)) return (int)0x80000000;
    return __float2int_rz (f);
}

struct Dr14State {
    float *emit_rms, *emit_peak; int* emit_valid;
    float *peak_hist, *m_rms, *m_peak, *m_dbtp;                // per channel (peak_hist: 2 per channel)
    unsigned long long* numfrag;                               // per instance
    uint32_t* phase;                                           // per instance: bank time of its last reset_peaks, mod the window length
    uint32_t* nwin;                                            // per instance: windows completed since its last reset_peaks (the window log's count)
    uint32_t* hist;                                            // [n_ch][8000]
    const float* cd;                                           // db_to_coeff ((b - 7999) / 100.0) for b = 0..7999, host libm
};

// The DR ports (:436-458) of an instance from its channels' top-20 % RMS scores m_rms and second-highest window peaks m_peak (dB):
// dr[c] = MIN (0, m_peak) - m_rms clamped to 1..20 (21: not yet valid), dr_total their average over the valid channels, clamped
// alike (21: none valid).  dr[1] is not written for a mono instance.
struct DrPorts { float dr[2], dr_total; };

B200M_DEV DrPorts dr_ports (const float* m_rms, const float* m_peak, int nch)
{
    DrPorts o;
    float dr_total = 0.0f; int dr_valid = 0;
#pragma unroll
    for (int c = 0; c < 2 && c < nch; ++c) {                  // unrolled: o stays in registers
        const float rdb = m_rms[c], pdb = m_peak[c];
        const float dr = __fsub_rn (0.0f < pdb ? 0.0f : pdb, rdb);                     // MIN (0, pdb) - rdb
        const bool ok = rdb > -80.0f && pdb > -80.0f;
        if (ok) { dr_total = __fadd_rn (dr_total, dr); ++dr_valid; }
        const float lo = 20.0f < dr ? 20.0f : dr;                                       // MAX (1, MIN (20, dr))
        o.dr[c] = ok ? (1.0f > lo ? 1.0f : lo) : 21.0f;
    }
    if (dr_valid > 0) { const float a = __fdiv_rn (dr_total, (float)dr_valid); const float lo = 20.0f < a ? 20.0f : a; o.dr_total = 1.0f > lo ? 1.0f : lo; }
    else o.dr_total = 21.0f;
    return o;
}

B200M_DEV float dr_block_count (unsigned long long num_fragments)      // 3.0 * num_fragments (:460)
{
    return __double2float_rn (__dmul_rn (3.0, (double)num_fragments));
}

// The window log (b200m_dr14_log_enable): a PointLog (common.cuh) of one b200m_dr14_point per completed 3 s window of an instance,
// planes [14][cap][n_inst] in the struct's field order.
constexpr int DR_LOG_FIELDS = 14;
static_assert (sizeof (b200m_dr14_point) == DR_LOG_FIELDS * sizeof (float), "b200m_dr14_point is 14 floats");

// Append instance inst's point for its window number win: rms / peak that window's own values per channel (dB), every other field
// from the instance's state after the window.  A mono instance's channel-1 fields and dr_total are NaN.
B200M_DEV void dr14_log_point (const PointLog& lg, int n_inst, int inst, int nch, const Dr14State& s, uint32_t win, bool silent,
                               float rms0, float rms1, float peak0, float peak1)
{
    const float nan = __int_as_float (0x7fc00000);
    const int ch0 = inst * nch;
    const DrPorts d = dr_ports (s.m_rms + ch0, s.m_peak + ch0, nch);
    const unsigned long long w = lg.written[inst];
    const size_t pl = (size_t)lg.cap * n_inst;
    float* p = lg.pts + (size_t)(w % lg.cap) * n_inst + inst;
    p[0] = (float)win;                                         // exact up to 2^24 windows
    p[pl] = silent ? 1.0f : 0.0f;
    p[2 * pl] = rms0; p[4 * pl] = peak0; p[6 * pl] = s.m_rms[ch0]; p[8 * pl] = s.m_peak[ch0]; p[10 * pl] = d.dr[0];
    if (nch > 1) { p[3 * pl] = rms1; p[5 * pl] = peak1; p[7 * pl] = s.m_rms[ch0 + 1]; p[9 * pl] = s.m_peak[ch0 + 1]; p[11 * pl] = d.dr[1]; p[12 * pl] = d.dr_total; }
    else { p[3 * pl] = nan; p[5 * pl] = nan; p[7 * pl] = nan; p[9 * pl] = nan; p[11 * pl] = nan; p[12 * pl] = nan; }
    p[13 * pl] = dr_block_count (s.numfrag[inst]);
    lg.written[inst] = w + 1;
}

// The mean of the loudest 20 % of the windows (:316-324): the bins of hist from the top down, 32 at a time by ballot, added in exactly
// the reference's bin order until m_cut windows are counted.  Called by the whole warp; the bins are read from L2 (__ldcg).  Returns
// the sum of cd^2 * count over the bins walked and their count in n_cut, the same in every lane.
B200M_DEV float dr_walk (const uint32_t* hist, const float* cd, uint32_t m_cut, int lane, uint32_t& n_cut)
{
    float rms_score = 0.0f;
    n_cut = 0;
    for (int base = DR_HISTBINS - 32; base >= 0 && n_cut < m_cut; base -= 32) {
        const int b = base + lane;
        const uint32_t bc = b > 0 ? __ldcg (&hist[b]) : 0u;
        unsigned mask = __ballot_sync (0xffffffffu, bc != 0);
        while (mask && n_cut < m_cut) {
            const int l = 31 - __clz (mask);
            const uint32_t bcl = __shfl_sync (0xffffffffu, bc, l);
            const float c = cd[base + l];
            rms_score = __fadd_rn (rms_score, __fmul_rn (__fmul_rn (c, c), (float)bcl));
            n_cut += bcl;
            mask &= ~(1u << l);
        }
    }
    return rms_score;
}

// dr14_calc_rms_score (:285-352) of the instances whose window closed in this block; one warp per instance.  With the window log
// on (lg.pts), lane 0 also appends the window's point.
// RAG: a ragged block, instance i ran over its first rlen[i] frames: its window closed only if the cut lies before that.
template <bool RAG = false>
__global__ void dr14_score_kernel (int n_inst, int nch, float n_sample_cnt_f, Dr14State s, TpkDr dr, int nfram, const uint32_t* __restrict__ rlen,
                                   PointLog lg)
{
    const int inst = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (inst >= n_inst) return;
    const int ch0 = inst * nch;
    const int cut = tpk_dr_cut (dr, inst, nfram);
    if (cut < 0) return;                                       // no window end in this block: emit_* still hold an older window's
    if (RAG && cut >= (int)rlen[inst]) return;                 // ... or none before the instance's last frame
    uint32_t win = 0;                                          // counted with the log off too: a log enabled later numbers windows alike
    if (lane == 0) { win = s.nwin[inst] + 1; s.nwin[inst] = win; }
    const float nan = __int_as_float (0x7fc00000);
    if (!s.emit_valid[ch0]) {                                  // silent window: nothing recorded (:287-297)
        // its RMS is logged as -80: what coeff_to_db gives for the RMS below 1e-4 that a sum <= 1e-9 n_sample_cnt means, and the
        // value for a window gated because its sum is NaN too.  Its peak is NaN: peak_cur carries on into the next window (:293-296).
        if (lg.pts && lane == 0) dr14_log_point (lg, n_inst, inst, nch, s, win, true, -80.0f, -80.0f, nan, nan);
        return;
    }
    unsigned long long nf = 0;
    if (lane == 0) { nf = s.numfrag[inst] + 1; s.numfrag[inst] = nf; }
    nf = __shfl_sync (0xffffffffu, nf, 0);
    const float mc = floorf (__double2float_rn (__ddiv_rn ((double)nf, 5.0)));      // MAX (1, floorf (num_fragments / 5.0)) (:301)
    const uint32_t m_cut = (uint32_t)(1.0f > mc ? 1.0f : mc);
    float wrms[2] = {nan, nan}, wpeak[2] = {nan, nan};         // lane 0: the window's own RMS and peak per channel, for the log
    for (int c = 0; c < nch; ++c) {
        const int ch = ch0 + c;
        uint32_t* hist = s.hist + (size_t)ch * DR_HISTBINS;
        if (lane == 0) {
            const float q = __fdiv_rn (__fmul_rn (2.0f, s.emit_rms[ch]), n_sample_cnt_f);
            const float rms = __double2float_rn (__dsqrt_rn ((double)q));                   // sqrt () in double (:304)
            const float rdb = dr_coeff_to_db (rms);
            if (c == 0) wrms[0] = rdb; else wrms[1] = rdb;
            int bin = dr_f2i (__fsub_rn (rintf (__fmul_rn (100.0f, __fadd_rn (80.0f, rdb))), 1.0f));   // (int)(rintf (..) - 1): float subtraction (:308)
            if (bin >= DR_HISTBINS) bin = DR_HISTBINS - 1;
            if (bin > 0) hist[bin] += 1;
        }
        __syncwarp ();
        uint32_t n_cut = 0; float rms_score = 0.0f;
        if (nf > 2) rms_score = dr_walk (hist, s.cd, m_cut, lane, n_cut);      // L2 reads: lane 0 has just incremented one bin
        if (lane == 0) {
            s.m_rms[ch] = n_cut > 0 ? dr_coeff_to_db (__fsqrt_rn (__fdiv_rn (rms_score, (float)n_cut))) : -81.0f;
            const float pc = s.emit_peak[ch];                  // second highest window peak (:339-351)
            if (c == 0) wpeak[0] = pc; else wpeak[1] = pc;
            float h0 = s.peak_hist[2 * ch], h1 = s.peak_hist[2 * ch + 1];
            if (pc >= h0) { h1 = h0; h0 = pc; } else if (pc > h1) h1 = pc;
            s.peak_hist[2 * ch] = h0; s.peak_hist[2 * ch + 1] = h1;
            s.m_peak[ch] = nf > 2 ? dr_coeff_to_db (h1) : -81.0f;
        }
        __syncwarp ();
    }
    if (lg.pts && lane == 0)
        dr14_log_point (lg, n_inst, inst, nch, s, win, false, wrms[0], wrms[1], dr_coeff_to_db (wpeak[0]), nch > 1 ? dr_coeff_to_db (wpeak[1]) : nan);
}

// read() results -> port values (:418-462); one thread per instance.  RAG: an instance with rlen 0 did not run (row and hold stay).
template <bool RAG = false>
__global__ void dr14_ports_kernel (int n_inst, int nch, int dr_mode, const b200m_tpk_result* __restrict__ res, Dr14State s,
                                   b200m_dr14_result* __restrict__ out, const uint32_t* __restrict__ rlen)
{
    const int inst = blockIdx.x * blockDim.x + threadIdx.x;
    if (inst >= n_inst) return;
    if (RAG && rlen[inst] == 0) return;
    b200m_dr14_result o;
    memset (&o, 0, sizeof (o));
    for (int c = 0; c < nch; ++c) {
        const int ch = inst * nch + c;
        const b200m_tpk_result r = res[ch];
        const float hold = s.m_dbtp[ch] > r.tp_p ? s.m_dbtp[ch] : r.tp_p;            // MAX (m_dbtp, pp)
        s.m_dbtp[ch] = hold;
        o.v_rms[c] = dr_coeff_to_db (r.km_rms);
        o.v_peak[c] = dr_coeff_to_db (r.tp_m);
        o.m_peak[c] = dr_coeff_to_db (hold);
        o.m_rms[c] = dr_mode ? s.m_rms[ch] : dr_coeff_to_db (r.km_peak);
    }
    if (dr_mode) {
        const DrPorts d = dr_ports (s.m_rms + inst * nch, s.m_peak + inst * nch, nch);
        o.dr[0] = d.dr[0];
        if (nch > 1) { o.dr[1] = d.dr[1]; o.dr_total = d.dr_total; }
    }
    o.block_count = dr_block_count (s.numfrag[inst]);
    out[inst] = o;
}

// a ragged block moves every instance's window clock on by its own length, not by the block's nfram: its phase (the bank time of
// its last reset, mod w) advances by nfram - rlen[i].  Queued behind the block's process() and scoring kernels, which read the old one.
__global__ void dr14_ragged_clock_kernel (int n_inst, const uint32_t* __restrict__ rlen, uint32_t nfram, uint32_t w, uint32_t* __restrict__ phase)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_inst) phase[i] = (phase[i] + (nfram - rlen[i]) % w) % w;
}

// reset_peaks (:246-262) of the instances inst[0 .. n_sel) (inst == nullptr: instances 0 .. n_sel - 1): their next window
// starts at bank time `tmod` (mod the window length).  The K-meter part is tpk_reset_inst.
__global__ void dr14_reset_kernel (const uint32_t* inst, size_t n_sel, int nch, int dr_mode, uint32_t tmod, float* rms_sum, float* peak_cur, Dr14State s)
{
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x, n_ch = n_sel * nch;
    auto chan = [&] (size_t k) { return inst ? (size_t)inst[k / nch] * nch + k % nch : k; };
    if (t < n_ch) { const size_t i = chan (t); s.m_peak[i] = -81.0f; s.m_rms[i] = -81.0f; s.m_dbtp[i] = 0.0f; rms_sum[i] = 0.0f; peak_cur[i] = 0.0f; s.peak_hist[2 * i] = 0.0f; s.peak_hist[2 * i + 1] = 0.0f; s.emit_valid[i] = 0; }
    if (t < n_sel) { const size_t j = inst ? inst[t] : t; s.numfrag[j] = 0; s.nwin[j] = 0; s.phase[j] = tmod; }
    if (dr_mode)
        for (size_t k = t; k < n_ch * DR_HISTBINS; k += (size_t)gridDim.x * blockDim.x) {
            if (!inst) { s.hist[k] = 0; continue; }
            const size_t r = k / DR_HISTBINS;
            s.hist[chan (r) * DR_HISTBINS + (k - r * DR_HISTBINS)] = 0;
        }
}

// Album DR (b200m_dr14_group_reduce / _finish).  The member list is the EBU bank's (GroupList, common.cuh): instances sorted by album,
// each member's album beside it, and each album's slice of the list.
//
// dr14_group_reduce_kernel: a 2-D grid of member chunks x column tiles.  CTA (x, y) takes DRG_CHUNK consecutive members of the list
// and DRG_TILE words of their histogram rows (an instance's nch x 8000 bins are contiguous: 16 B loads, coalesced); each thread keeps
// one uint4 of partial sums, DRG_BATCH members' loads in flight before their sums, and adds its non-zero sums into the album's
// zeroed row with integer atomicAdd when the album changes: order-independent, hence exact.  The histograms are sparse (a track
// fills a few dozen bins per channel), so the cost is the read.
constexpr int DRG_THREADS = 256, DRG_CHUNK = 16, DRG_BATCH = 4;
constexpr int DRG_TILE = DRG_THREADS * 4;                       // histogram words per column tile

__global__ void __launch_bounds__ (DRG_THREADS)
dr14_group_reduce_kernel (const uint32_t* __restrict__ hist, int row_words, const uint32_t* __restrict__ members,
                          const uint32_t* __restrict__ album, int n_members, int* __restrict__ rows)
{
    __shared__ uint32_t mem[DRG_CHUNK], alb[DRG_CHUNK];
    const int first = blockIdx.x * DRG_CHUNK, n = min (DRG_CHUNK, n_members - first);
    if (threadIdx.x < n) { mem[threadIdx.x] = members[first + threadIdx.x]; alb[threadIdx.x] = album[first + threadIdx.x]; }
    __syncthreads ();
    const int col = blockIdx.y * DRG_TILE + threadIdx.x * 4;
    if (col >= row_words) return;                               // row_words is a multiple of 4: a thread's 4 columns are all in
    const uint4* src = reinterpret_cast<const uint4*> (hist + col);
    const size_t pitch = (size_t)row_words / 4;
    uint4 acc = make_uint4 (0, 0, 0, 0);
    auto flush = [&] (uint32_t a) {
        int* row = rows + (size_t)a * (row_words + 2) + col;
        if (acc.x) atomicAdd (row, (int)acc.x);
        if (acc.y) atomicAdd (row + 1, (int)acc.y);
        if (acc.z) atomicAdd (row + 2, (int)acc.z);
        if (acc.w) atomicAdd (row + 3, (int)acc.w);
        acc = make_uint4 (0, 0, 0, 0);
    };
    uint32_t cur = alb[0];
    for (int k0 = 0; k0 < n; k0 += DRG_BATCH) {
        uint4 v[DRG_BATCH];
#pragma unroll
        for (int q = 0; q < DRG_BATCH; ++q)
            v[q] = k0 + q < n ? __ldcs (src + mem[k0 + q] * pitch) : make_uint4 (0, 0, 0, 0);      // read once: streaming loads
#pragma unroll
        for (int q = 0; q < DRG_BATCH; ++q) {
            if (k0 + q < n && alb[k0 + q] != cur) { flush (cur); cur = alb[k0 + q]; }           // uniform across the CTA
            acc.x += v[q].x; acc.y += v[q].y; acc.z += v[q].z; acc.w += v[q].w;
        }
    }
    flush (cur);
}

// The two largest of two top-two pairs (h0 >= h1, never NaN): the two largest of their union
struct Top2 { float h0, h1; };
B200M_DEV Top2 top2_merge (const Top2 a, const Top2 b)
{
    const bool ab = a.h0 >= b.h0;
    const float lo = ab ? b.h0 : a.h0, h1 = a.h1 >= b.h1 ? a.h1 : b.h1;
    return {ab ? a.h0 : b.h0, lo >= h1 ? lo : h1};
}

B200M_DEV Top2 top2_shfl_xor (const Top2 t, int o)
{
    return {__shfl_xor_sync (0xffffffffu, t.h0, o), __shfl_xor_sync (0xffffffffu, t.h1, o)};
}

// dr14_group_peaks_kernel: one warp per album walks its slice of the member list: the top two of the members' peak_hist pairs and
// the largest non-NaN m_dbtp per channel (fmaxf ignores NaN; an album without members holds 0), and the album's window and member
// counts, written into the last two words of its row.
constexpr int DRG_PEAK_WARPS = 8;

__global__ void __launch_bounds__ (DRG_PEAK_WARPS * 32)
dr14_group_peaks_kernel (int n_groups, int nch, const uint32_t* __restrict__ members, const uint32_t* __restrict__ off,
                         const float* __restrict__ peak_hist, const float* __restrict__ m_dbtp,
                         const unsigned long long* __restrict__ numfrag, int row_words, int* __restrict__ rows, float* __restrict__ peaks)
{
    const int lane = threadIdx.x & 31, g = blockIdx.x * DRG_PEAK_WARPS + (threadIdx.x >> 5);
    if (g >= n_groups) return;
    const uint32_t a = off[g], b = off[g + 1];
    const float nan = __int_as_float (0x7fc00000);
    Top2 t[2] = {{0.0f, 0.0f}, {0.0f, 0.0f}};
    float hold[2] = {nan, nan};
    unsigned long long nf = 0;
    for (uint32_t k = a + lane; k < b; k += 32) {
        const size_t m = members[k];
        nf += numfrag[m];
#pragma unroll
        for (int c = 0; c < 2; ++c)
            if (c < nch) {
                const size_t ch = m * nch + c;
                t[c] = top2_merge (t[c], {peak_hist[2 * ch], peak_hist[2 * ch + 1]});
                hold[c] = fmaxf (hold[c], m_dbtp[ch]);
            }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        nf += __shfl_xor_sync (0xffffffffu, nf, o);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            t[c] = top2_merge (t[c], top2_shfl_xor (t[c], o));
            hold[c] = fmaxf (hold[c], __shfl_xor_sync (0xffffffffu, hold[c], o));
        }
    }
    if (lane == 0) {
        int* tail = rows + (size_t)g * (row_words + 2) + row_words;
        tail[0] = (int)nf; tail[1] = (int)(b - a);
        for (int c = 0; c < nch; ++c) {
            float* p = peaks + ((size_t)g * nch + c) * 3;
            p[0] = t[c].h0; p[1] = t[c].h1; p[2] = b > a ? hold[c] : 0.0f;
        }
    }
}

// dr14_group_finish_kernel: one warp per (album, channel), DRG_FIN_ALBUMS albums per CTA.  The warp merges the n_parts peak blocks,
// then scores the channel's row as dr14_score_kernel scores an instance (dr_walk); lane 0 of an album's channel-0 warp applies the
// port arithmetic (dr_ports) to both channels.
constexpr int DRG_FIN_ALBUMS = 4;

__global__ void __launch_bounds__ (DRG_FIN_ALBUMS * 64)
dr14_group_finish_kernel (int n_groups, int nch, uint32_t n_parts, const int* rows, const float* __restrict__ peaks,
                          const float* __restrict__ cd, b200m_dr14_album* __restrict__ out)
{
    __shared__ float s_rms[DRG_FIN_ALBUMS][2], s_p2[DRG_FIN_ALBUMS][2], s_hold[DRG_FIN_ALBUMS][2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ga = warp / nch, c = warp % nch, g = blockIdx.x * DRG_FIN_ALBUMS + ga;
    const int row_words = nch * DR_HISTBINS;
    uint32_t nf = 0;
    if (g < n_groups) {
        const int* row = rows + (size_t)g * (row_words + 2);
        nf = (uint32_t)row[row_words];
        Top2 t = {0.0f, 0.0f};
        float hold = __int_as_float (0x7fc00000);
        for (uint32_t p = lane; p < n_parts; p += 32) {
            const float* q = peaks + (((size_t)p * n_groups + g) * nch + c) * 3;
            t = top2_merge (t, {q[0], q[1]});
            hold = fmaxf (hold, q[2]);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            t = top2_merge (t, top2_shfl_xor (t, o));
            hold = fmaxf (hold, __shfl_xor_sync (0xffffffffu, hold, o));
        }
        const float mc = floorf (__double2float_rn (__ddiv_rn ((double)nf, 5.0)));      // MAX (1, floorf (num_fragments / 5.0)) (:301)
        const uint32_t m_cut = (uint32_t)(1.0f > mc ? 1.0f : mc);
        uint32_t n_cut = 0; float rms_score = 0.0f;
        if (nf > 2) rms_score = dr_walk (reinterpret_cast<const uint32_t*> (row) + c * DR_HISTBINS, cd, m_cut, lane, n_cut);
        if (lane == 0) {
            s_rms[ga][c] = n_cut > 0 ? dr_coeff_to_db (__fsqrt_rn (__fdiv_rn (rms_score, (float)n_cut))) : -81.0f;
            s_p2[ga][c] = nf > 2 ? dr_coeff_to_db (t.h1) : -81.0f;
            s_hold[ga][c] = dr_coeff_to_db (hold);
        }
    }
    __syncthreads ();
    if (g >= n_groups || c != 0 || lane != 0) return;
    const float nan = __int_as_float (0x7fc00000);
    const DrPorts d = dr_ports (s_rms[ga], s_p2[ga], nch);
    b200m_dr14_album o;
    for (int k = 0; k < 2; ++k) {
        const bool on = k < nch;
        o.m_rms[k] = on ? s_rms[ga][k] : nan;
        o.peak2[k] = on ? s_p2[ga][k] : nan;
        o.dr[k] = on ? d.dr[k] : nan;
        o.m_peak[k] = on ? s_hold[ga][k] : nan;
    }
    o.dr_total = nch > 1 ? d.dr_total : nan;
    o.block_count = dr_block_count (nf);
    const int* tail = rows + (size_t)g * (row_words + 2) + row_words;
    o.windows = (float)nf; o.members = (float)(uint32_t)tail[1];
    out[g] = o;
}

}  // namespace b200m

using namespace b200m;

struct b200m_dr14 {
    int device; uint32_t n_inst, nch; double rate; int dr_mode;
    b200m_tpk* tpk = nullptr;
    uint64_t n_sample_cnt = 0;                                 // rintf (rate * 3.0) (:149)
    uint32_t w = 0, tmod = 0;                                  // window length n_sample_cnt + 1; bank sample clock mod w
    std::vector<uint32_t> phase;                               // host mirror of st.phase
    std::map<uint32_t, uint32_t> phases;                       // distinct phases -> number of instances on each
    uint32_t* d_sel = nullptr;                                 // instance list of a control call
    float *d_rms_sum = nullptr, *d_peak_cur = nullptr, *d_cd = nullptr;
    Dr14State st{}; b200m_dr14_result* d_out = nullptr;
    PointRing ring;                                            // the window log (b200m_dr14_log_enable), off while ring.log.pts is null
    GroupList grp;                                             // album DR (b200m_dr14_group_reduce): the member list
    b200m_dr14_album* d_alb = nullptr; uint32_t alb_cap = 0;   // the finish's device output, grown on demand
    BankPath path;
};

// reset_peaks of the instances d_inst[0 .. n_sel) (d_inst == nullptr: every instance), clear: and b200m_tpk_clear of their
// channels.  The host mirror of the phases is updated by the caller.
static int dr14_reset (b200m_dr14* h, const uint32_t* d_inst, uint32_t n_sel, bool clear, cudaStream_t st)
{
    const size_t n_ch = (size_t)n_sel * h->nch;
    dr14_reset_kernel<<<(unsigned)((n_ch + 255) / 256), 256, 0, st>>> (d_inst, n_sel, (int)h->nch, h->dr_mode, h->tmod, h->d_rms_sum, h->d_peak_cur, h->st);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return tpk_reset_inst (h->tpk, d_inst, n_sel, h->nch, clear, st);     // km[c]->reset () (:249)
}

static void dr14_set_phase (b200m_dr14* h, uint32_t inst, uint32_t p)
{
    auto it = h->phases.find (h->phase[inst]);
    if (--it->second == 0) h->phases.erase (it);
    h->phase[inst] = p;
    ++h->phases[p];
}

// does some instance's window close in the next block of nfram samples?  Phase p closes at block sample (p - tmod - 1) mod w.
static bool dr14_closes (const b200m_dr14* h, uint32_t nfram)
{
    const uint32_t a = (h->tmod + 1) % h->w, b = a + nfram;   // phases in [a, b), taken mod w
    auto it = h->phases.lower_bound (a);
    if (it != h->phases.end () && it->first < b) return true;
    return b > h->w && h->phases.begin ()->first < b - h->w;
}

// len (host, every entry <= nfram, some != nfram: ragged_check): a ragged block, instance i runs over its first len[i] frames;
// nullptr: every instance runs nfram
static int dr14_run (b200m_dr14* h, const float* d_in, size_t stride, uint32_t nfram, cudaStream_t st, const uint32_t* len = nullptr)
{
    // a ragged block: per-instance lengths and K-meter _fall values, uploaded through the true-peak bank's staging and _fall cache
    const uint32_t* d_len = nullptr; const float* d_fall = nullptr;
    if (len) if (int rc = tpk_upload_len (h->tpk, len, h->n_inst, st, &d_len, &d_fall)) return rc;
    bool closes = false;
    TpkDr dr = {};
    if (h->dr_mode) {
        closes = dr14_closes (h, nfram);
        dr = {h->d_rms_sum, h->d_peak_cur, h->st.emit_rms, h->st.emit_peak, h->st.emit_valid, h->st.phase, h->tmod, h->w, (int)h->nch,
              1e-9 * (double)(float)h->n_sample_cnt};
        tpk_set_dr (h->tpk, &dr);
        h->tmod = (uint32_t)((h->tmod + (uint64_t)nfram) % h->w);
    }
    int rc = len ? tpk_process_ragged (h->tpk, d_in, stride, nfram, st, d_len, d_fall, h->nch)
                 : b200m_tpk_process_device (h->tpk, d_in, stride, nfram, B200M_TP_MODE_PROCESS, st);
    if (rc) return rc;
    const unsigned gs = (h->n_inst * 32 + 127) / 128, gp = (h->n_inst + 127) / 128;
    if (closes) {
        if (len) dr14_score_kernel<true><<<gs, 128, 0, st>>> ((int)h->n_inst, (int)h->nch, (float)h->n_sample_cnt, h->st, dr, (int)nfram, d_len, h->ring.log);
        else dr14_score_kernel<<<gs, 128, 0, st>>> ((int)h->n_inst, (int)h->nch, (float)h->n_sample_cnt, h->st, dr, (int)nfram, nullptr, h->ring.log);
        B200M_LAUNCHED (1);
    }
    if ((rc = len ? tpk_read_ragged (h->tpk, st, d_len, h->nch) : b200m_tpk_read_device (h->tpk, st))) return rc;
    if (len) dr14_ports_kernel<true><<<gp, 128, 0, st>>> ((int)h->n_inst, (int)h->nch, h->dr_mode, tpk_device_results (h->tpk), h->st, h->d_out, d_len);
    else dr14_ports_kernel<<<gp, 128, 0, st>>> ((int)h->n_inst, (int)h->nch, h->dr_mode, tpk_device_results (h->tpk), h->st, h->d_out, nullptr);
    B200M_LAUNCHED (1);
    if (len && h->dr_mode) {
        // each instance's clock ran len[i] frames: move the phases on the device and in the host mirror
        dr14_ragged_clock_kernel<<<gp, 128, 0, st>>> ((int)h->n_inst, d_len, nfram, h->w, h->st.phase);
        B200M_LAUNCHED (1);
        for (uint32_t i = 0; i < h->n_inst; ++i)
            if (len[i] != nfram) dr14_set_phase (h, i, (h->phase[i] + (nfram - len[i]) % h->w) % h->w);
    }
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

extern "C" {

int b200m_dr14_create (b200m_dr14** out, int device, uint32_t n_inst, uint32_t n_channels, double rate, int dr_mode)
{
    if (!out) return set_err (B200M_E_INVAL, "NULL out pointer");
    *out = nullptr;
    if (n_inst == 0 || n_channels < 1 || n_channels > 2 || !(rate >= 1000.0)) return set_err (B200M_E_INVAL, "bad n_inst/n_channels/rate");
    if (dr_mode && rintf ((float)(rate * 3.0)) < (float)B200M_MAX_BLOCK)
        return set_err (B200M_E_UNSUPPORTED, "DR mode needs a 3 s window longer than the largest block (rate >= %d Hz)", B200M_MAX_BLOCK / 3 + 1);
    b200m_dr14* h = new (std::nothrow) b200m_dr14;
    if (!h) return set_err (B200M_E_NOMEM, "host allocation failed");
    h->device = device; h->n_inst = n_inst; h->nch = n_channels; h->rate = rate; h->dr_mode = dr_mode ? 1 : 0;
    h->n_sample_cnt = (uint64_t)rintf ((float)(rate * 3.0));   // n_sample_cnt = rintf (rate * 3.0) (:149)
    h->w = (uint32_t)(h->n_sample_cnt + 1);                    // "if (++scnt > slmt)" (:411): a window every n_sample_cnt + 1 samples
    h->phase.assign (n_inst, 0);
    h->phases[0] = n_inst;
    const size_t n_ch = (size_t)n_inst * n_channels;
    int rc = b200m_tpk_create (&h->tpk, device, (uint32_t)n_ch, (float)rate, B200M_TPK_TRUEPEAK | B200M_TPK_KMETER);
    if (rc) { delete h; return rc; }
    DeviceGuard g (device);
    cudaError_t e = cudaSuccess;
    auto A = [&] (void** p, size_t bytes) { if (e == cudaSuccess) { e = cudaMalloc (p, bytes); if (e == cudaSuccess) e = cudaMemset (*p, 0, bytes); } };
    A ((void**)&h->d_rms_sum, n_ch * 4); A ((void**)&h->d_peak_cur, n_ch * 4);
    A ((void**)&h->st.emit_rms, n_ch * 4); A ((void**)&h->st.emit_peak, n_ch * 4); A ((void**)&h->st.emit_valid, n_ch * 4);
    A ((void**)&h->st.peak_hist, n_ch * 8); A ((void**)&h->st.m_rms, n_ch * 4); A ((void**)&h->st.m_peak, n_ch * 4); A ((void**)&h->st.m_dbtp, n_ch * 4);
    A ((void**)&h->st.numfrag, (size_t)n_inst * 8); A ((void**)&h->st.phase, (size_t)n_inst * 4); A ((void**)&h->st.nwin, (size_t)n_inst * 4); A ((void**)&h->d_sel, (size_t)n_inst * 4);
    if (h->dr_mode) A ((void**)&h->st.hist, n_ch * DR_HISTBINS * 4);
    A ((void**)&h->d_cd, DR_HISTBINS * 4); A ((void**)&h->d_out, (size_t)n_inst * sizeof (b200m_dr14_result));
    if (e == cudaSuccess) {
        // db_to_coeff ((b - DR_HISTBINS + 1) / 100.0) (:241-244,319) with the host libm, expression types as in the reference
        float* cd = (float*)malloc (DR_HISTBINS * sizeof (float));
        if (!cd) e = cudaErrorMemoryAllocation;
        else {
            for (int b = 0; b < DR_HISTBINS; ++b) { const float db = (b - DR_HISTBINS + 1) / 100.0; cd[b] = db <= -80 ? 0.0f : powf (10, 0.05 * db); }
            e = cudaMemcpy (h->d_cd, cd, DR_HISTBINS * sizeof (float), cudaMemcpyHostToDevice);
            free (cd);
        }
        h->st.cd = h->d_cd;
    }
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags (&h->path.own, cudaStreamNonBlocking);
    if (e == cudaSuccess) {                                    // instantiate: m_rms = m_peak = -81 (:157-158)
        dr14_reset_kernel<<<(unsigned)((n_ch + 255) / 256), 256>>> (nullptr, n_inst, (int)n_channels, h->dr_mode, 0u, h->d_rms_sum, h->d_peak_cur, h->st);
        B200M_LAUNCHED (1);
        e = cudaDeviceSynchronize ();
    }
    if (e != cudaSuccess) { rc = cuda_fail (e, "dr14_create", __FILE__, __LINE__); b200m_dr14_destroy (h); return rc; }
    *out = h;
    return 0;
}

int b200m_dr14_destroy (b200m_dr14* h)
{
    if (!h) return 0;
    b200m_tpk_destroy (h->tpk);
    DeviceGuard g (h->device);
    cudaDeviceSynchronize ();
    void* ps[] = {h->d_rms_sum, h->d_peak_cur, h->st.emit_rms, h->st.emit_peak, h->st.emit_valid, h->st.peak_hist, h->st.m_rms, h->st.m_peak,
                  h->st.m_dbtp, h->st.numfrag, h->st.phase, h->st.nwin, h->d_sel, h->st.hist, h->d_cd, h->d_out};
    for (void* p : ps) cudaFree (p);
    h->ring.release ();
    h->grp.release (); cudaFree (h->d_alb);
    h->path.release ();
    delete h;
    return 0;
}

// every block entry point: one stream for the copy and every kernel, the true-peak bank driven on its device path on that stream
static int dr14_block (b200m_dr14* h, const float* in, size_t stride, uint32_t nfram, bool host, void* stream, const uint32_t* len)
{
    return bank_call (h, in, stride, nfram, host, stream, h ? (size_t)h->n_inst * h->nch : 0, h ? h->n_inst : 0, len, no_check,
                      [&] (const float* d_in, size_t ds, cudaStream_t st, const uint32_t* rlen) { return dr14_run (h, d_in, ds, nfram, st, rlen); });
}

int b200m_dr14_run_device (b200m_dr14* h, const float* d_in, size_t stride, uint32_t nfram, void* stream)
{
    return dr14_block (h, d_in, stride, nfram, false, stream, nullptr);
}

int b200m_dr14_run_host (b200m_dr14* h, const float* in, size_t stride, uint32_t nfram)
{
    return dr14_block (h, in, stride, nfram, true, nullptr, nullptr);
}

int b200m_dr14_run_ragged_device (b200m_dr14* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream)
{
    return dr14_block (h, d_in, stride, nfram, false, stream, len);
}

int b200m_dr14_run_ragged_host (b200m_dr14* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len)
{
    return dr14_block (h, in, stride, nfram, true, nullptr, len);
}

int b200m_dr14_reset (b200m_dr14* h, void* stream)              // reset_peaks (:241-258), every instance
{
    return b200m_dr14_control (h, nullptr, 0, B200M_DR14_RESET, stream);
}

int b200m_dr14_control (b200m_dr14* h, const uint32_t* inst, uint32_t count, int cmd, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    if (cmd != B200M_DR14_RESET && cmd != B200M_DR14_CLEAR) return set_err (B200M_E_INVAL, "unknown control %d", cmd);
    if (!inst && count) return set_err (B200M_E_INVAL, "NULL instance list");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    if (!inst) {
        h->phase.assign (h->n_inst, h->tmod);
        h->phases.clear (); h->phases[h->tmod] = h->n_inst;
        return dr14_reset (h, nullptr, h->n_inst, cmd == B200M_DR14_CLEAR, st);
    }
    std::vector<uint32_t> sel;                                 // the listed instances, each once
    std::vector<uint8_t> seen (h->n_inst, 0);
    for (uint32_t k = 0; k < count; ++k) {
        if (inst[k] >= h->n_inst) return set_err (B200M_E_INVAL, "bad instance %u", inst[k]);
        if (!seen[inst[k]]) { seen[inst[k]] = 1; sel.push_back (inst[k]); }
    }
    if (sel.empty ()) return 0;
    B200M_CUDA (cudaMemcpyAsync (h->d_sel, sel.data (), sel.size () * sizeof (uint32_t), cudaMemcpyHostToDevice, st));
    for (uint32_t i : sel) dr14_set_phase (h, i, h->tmod);
    return dr14_reset (h, h->d_sel, (uint32_t)sel.size (), cmd == B200M_DR14_CLEAR, st);
}

int b200m_dr14_results (b200m_dr14* h, b200m_dr14_result* out, void* stream)
{
    if (!h || !out) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    B200M_CUDA (cudaMemcpyAsync (out, h->d_out, (size_t)h->n_inst * sizeof (b200m_dr14_result), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_dr14_histogram (b200m_dr14* h, uint32_t inst, uint32_t chan, uint32_t* hist8000, void* stream)
{
    if (!h || !hist8000 || inst >= h->n_inst || chan >= h->nch || !h->dr_mode) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    B200M_CUDA (cudaMemcpyAsync (hist8000, h->st.hist + ((size_t)inst * h->nch + chan) * DR_HISTBINS, DR_HISTBINS * 4, cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_dr14_log_enable (b200m_dr14* h, uint32_t capacity, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    if (!h->dr_mode) return set_err (B200M_E_UNSUPPORTED, "a TPnRMS bank has no 3 s windows to log");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    if (h->ring.log.pts) {                                     // kernels in flight may still write the old log
        B200M_CUDA (cudaStreamSynchronize (st));
        h->ring.release ();
    }
    if (capacity == 0) return 0;
    const cudaError_t e = h->ring.alloc (h->n_inst, capacity, DR_LOG_FIELDS, st);
    if (e != cudaSuccess) {
        cudaGetLastError ();                                   // a failed allocation is not sticky: later calls must not see it
        if (e == cudaErrorMemoryAllocation) return set_err (B200M_E_NOMEM, "window log of %u points x %u instances: out of device memory", capacity, h->n_inst);
        return cuda_fail (e, "b200m_dr14_log_enable", __FILE__, __LINE__);
    }
    return 0;
}

uint32_t b200m_dr14_log_capacity (const b200m_dr14* h)
{
    return h ? h->ring.log.cap : 0;
}

int b200m_dr14_log_drain (b200m_dr14* h, b200m_dr14_point* out, uint32_t* count, uint64_t* lost, void* stream)
{
    if (!h || !out || !count || !lost) return set_err (B200M_E_INVAL, "NULL argument");
    if (!h->ring.log.pts) return set_err (B200M_E_INVAL, "the window log is off (b200m_dr14_log_enable)");
    DeviceGuard g (h->device);
    // 16 points per tile: the drain's static tile of 32 x (16 x 14 + 1) floats stays under 48 KB
    return log_drain<DR_LOG_FIELDS, 16> (h->ring, h->n_inst, (float*)out, count, lost, h->path.stream (stream));
}

int b200m_dr14_group_reduce (b200m_dr14* h, const uint32_t* group, uint32_t n_groups, int32_t* d_rows, float* d_peaks, void* stream)
{
    if (!h || !group || !d_rows || !d_peaks) return set_err (B200M_E_INVAL, "NULL argument");
    if (!h->dr_mode) return set_err (B200M_E_UNSUPPORTED, "a TPnRMS bank has no window histograms to pool");
    if (int rc = group_check (group, h->n_inst, n_groups, B200M_DR14_MAX_GROUPS)) return rc;
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    if (int rc = h->grp.assign (group, h->n_inst, n_groups, B200M_DR14_MAX_GROUPS, st)) return rc;
    const uint32_t nm = h->grp.members, rw = h->nch * DR_HISTBINS;
    B200M_CUDA (cudaMemsetAsync (d_rows, 0, (size_t)n_groups * (rw + 2) * sizeof (int32_t), st));
    if (nm) {
        const dim3 grid ((nm + DRG_CHUNK - 1) / DRG_CHUNK, (rw + DRG_TILE - 1) / DRG_TILE);
        dr14_group_reduce_kernel<<<grid, DRG_THREADS, 0, st>>> (h->st.hist, (int)rw, h->grp.d_members (), h->grp.d_album (), (int)nm, d_rows);
        B200M_LAUNCHED (1);
    }
    dr14_group_peaks_kernel<<<(n_groups + DRG_PEAK_WARPS - 1) / DRG_PEAK_WARPS, DRG_PEAK_WARPS * 32, 0, st>>> (
        (int)n_groups, (int)h->nch, h->grp.d_members (), h->grp.d_off (), h->st.peak_hist, h->st.m_dbtp, h->st.numfrag, (int)rw, d_rows, d_peaks);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

int b200m_dr14_group_finish (b200m_dr14* h, const int32_t* d_rows, const float* d_peaks, uint32_t n_parts, uint32_t n_groups,
                             b200m_dr14_album* out, void* stream)
{
    if (!h || !d_rows || !d_peaks || !out) return set_err (B200M_E_INVAL, "NULL argument");
    if (!h->dr_mode) return set_err (B200M_E_UNSUPPORTED, "a TPnRMS bank has no window histograms to pool");
    if (n_groups == 0 || n_groups > B200M_DR14_MAX_GROUPS) return set_err (B200M_E_INVAL, "n_groups %u outside 1..%u", n_groups, B200M_DR14_MAX_GROUPS);
    if (n_parts == 0) return set_err (B200M_E_INVAL, "n_parts is 0");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    if (n_groups > h->alb_cap) {                               // the previous call synchronised: nothing in flight uses the old buffer
        cudaFree (h->d_alb); h->d_alb = nullptr; h->alb_cap = 0;
        if (cudaMalloc ((void**)&h->d_alb, (size_t)n_groups * sizeof (b200m_dr14_album)) != cudaSuccess) {
            cudaGetLastError ();
            return set_err (B200M_E_NOMEM, "album results of %u groups: out of device memory", n_groups);
        }
        h->alb_cap = n_groups;
    }
    dr14_group_finish_kernel<<<(n_groups + DRG_FIN_ALBUMS - 1) / DRG_FIN_ALBUMS, DRG_FIN_ALBUMS * 32 * h->nch, 0, st>>> (
        (int)n_groups, (int)h->nch, n_parts, d_rows, d_peaks, h->d_cd, h->d_alb);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    B200M_CUDA (cudaMemcpyAsync (out, h->d_alb, (size_t)n_groups * sizeof (b200m_dr14_album), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

}  // extern "C"
