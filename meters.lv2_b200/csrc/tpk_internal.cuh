// tpk_internal.cuh — pieces of the true-peak / K-meter bank (tpk.cu) shared with the DR-14 bank (dr14.cu).
#pragma once
#include "common.cuh"

namespace b200m {

// DR-14 accumulation riding on the process() kernel (dr14_run's sample loop, src/dr14.c:401-416): per channel
// rms_sum += v * v; peak_cur = MAX (peak_cur, v); when an instance's 3 s window closes inside this block the sums are handed
// to the scoring kernel (dr14.cu) unless the whole instance was silent (dr14_calc_rms_score :287-297).  rms_sum == nullptr: off.
// Every instance has its own window phase (the bank time of its last reset, mod w); the process kernels only read it, so a
// kernel that runs several times per block (the slab pipeline) needs no clock of its own.
struct TpkDr {
    float *rms_sum, *peak_cur;              // running, per channel
    float *emit_rms, *emit_peak; int* emit_valid;      // the closed window's values, per channel; valid = 0 for a silent instance
    const uint32_t* phase;                  // per instance: bank time of its last reset, mod w
    uint32_t tmod, w;                       // bank time of this block's first sample, mod w; w = n_sample_cnt + 1 (window length)
    int nch;                                // channels per instance
    double silent_thr;                      // 1e-9 * (float) n_sample_cnt
};

// "if (++scnt > slmt)" (:410) of instance `inst`: the sample of this block after which its window closes, or -1.  Windows end at
// bank times t with t = phase + w - 1 (mod w); w > B200M_MAX_BLOCK, so at most one falls in a block.
B200M_DEV int tpk_dr_cut (const TpkDr& dr, int inst, int nfram)
{
    uint32_t j = dr.phase[inst] + dr.w - 1u - dr.tmod;
    if (j >= dr.w) j -= dr.w;
    return j < (uint32_t)nfram ? (int)j : -1;
}

// internal hooks of the true-peak / K-meter bank for dr14.cu (hidden visibility)
void tpk_set_dr (b200m_tpk* h, const TpkDr* dr);                 // DR accumulation of the following process() calls (nullptr: off)
const b200m_tpk_result* tpk_device_results (b200m_tpk* h);      // device array filled by b200m_tpk_read_device
// Kmeterdsp::reset (clear: b200m_tpk_clear) of the channels d_inst[k] * per .. + per - 1, k < n_sel (d_inst == nullptr: every channel)
int tpk_reset_inst (b200m_tpk* h, const uint32_t* d_inst, uint32_t n_sel, uint32_t per, bool clear, cudaStream_t st);
// Kmeterdsp's _fall for a process() call of n frames, computed with the host libm as the reference does (kmeterdsp.cc:65-70)
float tpk_km_fall (const b200m_tpk* h, uint32_t n);
// Enqueue on `st` the upload of n <= n_chan lengths and their K-meter _fall values (tpk_km_fall, cached per length) through the
// bank's pinned staging; *d_len and *d_fall are the device arrays the following kernels on `st` read.
int tpk_upload_len (b200m_tpk* h, const uint32_t* len, uint32_t n, cudaStream_t st, const uint32_t** d_len, const float** d_fall);
// A ragged process() block (with the DR accumulation set by tpk_set_dr): channel c belongs to instance c / per, which processes its
// first d_len[c / per] <= nfram frames; d_fall[c / per] = tpk_km_fall (that length).  Length 0: the channel is not touched.  Always
// the exact kernel, also in tolerance mode.  Device arrays, read by the kernels queued on `st`.
int tpk_process_ragged (b200m_tpk* h, const float* d_in, size_t stride, uint32_t nfram, cudaStream_t st, const uint32_t* d_len,
                        const float* d_fall, uint32_t per);
// b200m_tpk_read_device after a ragged block: the channels of instances with d_len 0 are not read
int tpk_read_ragged (b200m_tpk* h, cudaStream_t st, const uint32_t* d_len, uint32_t per);

}  // namespace b200m
