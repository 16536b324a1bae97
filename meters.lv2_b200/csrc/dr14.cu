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
    uint32_t* hist;                                            // [n_ch][8000]
    const float* cd;                                           // db_to_coeff ((b - 7999) / 100.0) for b = 0..7999, host libm
};

// dr14_calc_rms_score (:285-352) of the instances whose window closed in this block; one warp per instance
__global__ void dr14_score_kernel (int n_inst, int nch, float n_sample_cnt_f, Dr14State s, TpkDr dr, int nfram)
{
    const int inst = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (inst >= n_inst) return;
    const int ch0 = inst * nch;
    if (tpk_dr_cut (dr, inst, nfram) < 0) return;             // no window end in this block: emit_* still hold an older window's
    if (!s.emit_valid[ch0]) return;                            // silent window: nothing recorded (:287-297)
    unsigned long long nf = 0;
    if (lane == 0) { nf = s.numfrag[inst] + 1; s.numfrag[inst] = nf; }
    nf = __shfl_sync (0xffffffffu, nf, 0);
    const float mc = floorf (__double2float_rn (__ddiv_rn ((double)nf, 5.0)));      // MAX (1, floorf (num_fragments / 5.0)) (:301)
    const uint32_t m_cut = (uint32_t)(1.0f > mc ? 1.0f : mc);
    for (int c = 0; c < nch; ++c) {
        const int ch = ch0 + c;
        uint32_t* hist = s.hist + (size_t)ch * DR_HISTBINS;
        if (lane == 0) {
            const float q = __fdiv_rn (__fmul_rn (2.0f, s.emit_rms[ch]), n_sample_cnt_f);
            const float rms = __double2float_rn (__dsqrt_rn ((double)q));                   // sqrt () in double (:304)
            int bin = dr_f2i (__fsub_rn (rintf (__fmul_rn (100.0f, __fadd_rn (80.0f, dr_coeff_to_db (rms)))), 1.0f));   // (int)(rintf (..) - 1): float subtraction (:308)
            if (bin >= DR_HISTBINS) bin = DR_HISTBINS - 1;
            if (bin > 0) hist[bin] += 1;
        }
        __syncwarp ();
        uint32_t n_cut = 0; float rms_score = 0.0f;
        if (nf > 2) {                                          // mean of the loudest 20 % (:316-324), bins in descending order
            for (int base = DR_HISTBINS - 32; base >= 0 && n_cut < m_cut; base -= 32) {
                const int b = base + lane;
                const uint32_t bc = b > 0 ? __ldcg (&hist[b]) : 0u;      // L2 read: lane 0 has just incremented one bin
                unsigned mask = __ballot_sync (0xffffffffu, bc != 0);
                while (mask && n_cut < m_cut) {
                    const int l = 31 - __clz (mask);
                    const uint32_t bcl = __shfl_sync (0xffffffffu, bc, l);
                    const float cd = s.cd[base + l];
                    rms_score = __fadd_rn (rms_score, __fmul_rn (__fmul_rn (cd, cd), (float)bcl));
                    n_cut += bcl;
                    mask &= ~(1u << l);
                }
            }
        }
        if (lane == 0) {
            s.m_rms[ch] = n_cut > 0 ? dr_coeff_to_db (__fsqrt_rn (__fdiv_rn (rms_score, (float)n_cut))) : -81.0f;
            const float pc = s.emit_peak[ch];                  // second highest window peak (:339-351)
            float h0 = s.peak_hist[2 * ch], h1 = s.peak_hist[2 * ch + 1];
            if (pc >= h0) { h1 = h0; h0 = pc; } else if (pc > h1) h1 = pc;
            s.peak_hist[2 * ch] = h0; s.peak_hist[2 * ch + 1] = h1;
            s.m_peak[ch] = nf > 2 ? dr_coeff_to_db (h1) : -81.0f;
        }
        __syncwarp ();
    }
}

// read() results -> port values (:418-462); one thread per instance
__global__ void dr14_ports_kernel (int n_inst, int nch, int dr_mode, const b200m_tpk_result* __restrict__ res, Dr14State s,
                                   b200m_dr14_result* __restrict__ out)
{
    const int inst = blockIdx.x * blockDim.x + threadIdx.x;
    if (inst >= n_inst) return;
    b200m_dr14_result o;
    memset (&o, 0, sizeof (o));
    float dr_total = 0.0f; int dr_valid = 0;
    for (int c = 0; c < nch; ++c) {
        const int ch = inst * nch + c;
        const b200m_tpk_result r = res[ch];
        const float hold = s.m_dbtp[ch] > r.tp_p ? s.m_dbtp[ch] : r.tp_p;            // MAX (m_dbtp, pp)
        s.m_dbtp[ch] = hold;
        o.v_rms[c] = dr_coeff_to_db (r.km_rms);
        o.v_peak[c] = dr_coeff_to_db (r.tp_m);
        o.m_peak[c] = dr_coeff_to_db (hold);
        if (dr_mode) {
            const float rdb = s.m_rms[ch], pdb = s.m_peak[ch];
            const float dr = __fsub_rn (0.0f < pdb ? 0.0f : pdb, rdb);                 // MIN (0, pdb) - rdb
            const bool ok = rdb > -80.0f && pdb > -80.0f;
            if (ok) { dr_total = __fadd_rn (dr_total, dr); ++dr_valid; }
            const float lo = 20.0f < dr ? 20.0f : dr;                                   // MAX (1, MIN (20, dr))
            o.dr[c] = ok ? (1.0f > lo ? 1.0f : lo) : 21.0f;
            o.m_rms[c] = rdb;
        } else o.m_rms[c] = dr_coeff_to_db (r.km_peak);
    }
    if (nch > 1 && dr_mode) {
        if (dr_valid > 0) { const float a = __fdiv_rn (dr_total, (float)dr_valid); const float lo = 20.0f < a ? 20.0f : a; o.dr_total = 1.0f > lo ? 1.0f : lo; }
        else o.dr_total = 21.0f;
    }
    o.block_count = __double2float_rn (__dmul_rn (3.0, (double)s.numfrag[inst]));     // 3.0 * num_fragments
    out[inst] = o;
}

// reset_peaks (:246-262) of the instances inst[0 .. n_sel) (inst == nullptr: instances 0 .. n_sel - 1): their next window
// starts at bank time `tmod` (mod the window length).  The K-meter part is tpk_reset_inst.
__global__ void dr14_reset_kernel (const uint32_t* inst, size_t n_sel, int nch, int dr_mode, uint32_t tmod, float* rms_sum, float* peak_cur, Dr14State s)
{
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x, n_ch = n_sel * nch;
    auto chan = [&] (size_t k) { return inst ? (size_t)inst[k / nch] * nch + k % nch : k; };
    if (t < n_ch) { const size_t i = chan (t); s.m_peak[i] = -81.0f; s.m_rms[i] = -81.0f; s.m_dbtp[i] = 0.0f; rms_sum[i] = 0.0f; peak_cur[i] = 0.0f; s.peak_hist[2 * i] = 0.0f; s.peak_hist[2 * i + 1] = 0.0f; s.emit_valid[i] = 0; }
    if (t < n_sel) { const size_t j = inst ? inst[t] : t; s.numfrag[j] = 0; s.phase[j] = tmod; }
    if (dr_mode)
        for (size_t k = t; k < n_ch * DR_HISTBINS; k += (size_t)gridDim.x * blockDim.x) {
            if (!inst) { s.hist[k] = 0; continue; }
            const size_t r = k / DR_HISTBINS;
            s.hist[chan (r) * DR_HISTBINS + (k - r * DR_HISTBINS)] = 0;
        }
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
    cudaStream_t own = nullptr; HostStage stage; bool last_host = false;
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

static int dr14_run (b200m_dr14* h, const float* d_in, size_t stride, uint32_t nfram, cudaStream_t st)
{
    bool closes = false;
    TpkDr dr = {};
    if (h->dr_mode) {
        closes = dr14_closes (h, nfram);
        dr = {h->d_rms_sum, h->d_peak_cur, h->st.emit_rms, h->st.emit_peak, h->st.emit_valid, h->st.phase, h->tmod, h->w, (int)h->nch,
              1e-9 * (double)(float)h->n_sample_cnt};
        tpk_set_dr (h->tpk, &dr);
        h->tmod = (uint32_t)((h->tmod + (uint64_t)nfram) % h->w);
    }
    int rc = b200m_tpk_process_device (h->tpk, d_in, stride, nfram, B200M_TP_MODE_PROCESS, st);
    if (rc) return rc;
    if (closes) {
        dr14_score_kernel<<<(h->n_inst * 32 + 127) / 128, 128, 0, st>>> ((int)h->n_inst, (int)h->nch, (float)h->n_sample_cnt, h->st, dr, (int)nfram);
        B200M_LAUNCHED (1);
    }
    if ((rc = b200m_tpk_read_device (h->tpk, st))) return rc;
    dr14_ports_kernel<<<(h->n_inst + 127) / 128, 128, 0, st>>> ((int)h->n_inst, (int)h->nch, h->dr_mode, tpk_device_results (h->tpk), h->st, h->d_out);
    B200M_LAUNCHED (1);
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
    A ((void**)&h->st.numfrag, (size_t)n_inst * 8); A ((void**)&h->st.phase, (size_t)n_inst * 4); A ((void**)&h->d_sel, (size_t)n_inst * 4);
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
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags (&h->own, cudaStreamNonBlocking);
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
                  h->st.m_dbtp, h->st.numfrag, h->st.phase, h->d_sel, h->st.hist, h->d_cd, h->d_out};
    for (void* p : ps) cudaFree (p);
    h->stage.release ();
    if (h->own) cudaStreamDestroy (h->own);
    delete h;
    return 0;
}

int b200m_dr14_run_device (b200m_dr14* h, const float* d_in, size_t stride, uint32_t nfram, void* stream)
{
    if (int rc = check_block_args (h, d_in, stride, nfram)) return rc;
    DeviceGuard g (h->device);
    h->last_host = false;
    return dr14_run (h, d_in, stride, nfram, (cudaStream_t)stream);
}

int b200m_dr14_run_host (b200m_dr14* h, const float* in, size_t stride, uint32_t nfram)
{
    if (int rc = check_block_args (h, in, stride, nfram)) return rc;
    DeviceGuard g (h->device);
    B200M_ENTER_HOST_PATH (h);
    // one stream for the copy and every kernel: stage here, then drive the true-peak bank's device path on it
    const size_t n_ch = (size_t)h->n_inst * h->nch;
    if (h->stage.ensure (n_ch, nfram)) return set_err (B200M_E_NOMEM, "staging buffer allocation failed");
    B200M_CUDA (cudaMemcpy2DAsync (h->stage.d, h->stage.cap * sizeof (float), in, stride * sizeof (float), (size_t)nfram * sizeof (float), n_ch,
                                   cudaMemcpyHostToDevice, h->own));
    h->last_host = true;
    return dr14_run (h, h->stage.d, h->stage.cap, nfram, h->own);
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
    cudaStream_t st = h->last_host ? h->own : (cudaStream_t)stream;
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
    cudaStream_t st = h->last_host ? h->own : (cudaStream_t)stream;
    B200M_CUDA (cudaMemcpyAsync (out, h->d_out, (size_t)h->n_inst * sizeof (b200m_dr14_result), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_dr14_histogram (b200m_dr14* h, uint32_t inst, uint32_t chan, uint32_t* hist8000, void* stream)
{
    if (!h || !hist8000 || inst >= h->n_inst || chan >= h->nch || !h->dr_mode) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->last_host ? h->own : (cudaStream_t)stream;
    B200M_CUDA (cudaMemcpyAsync (hist8000, h->st.hist + ((size_t)inst * h->nch + chan) * DR_HISTBINS, DR_HISTBINS * 4, cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

}  // extern "C"
