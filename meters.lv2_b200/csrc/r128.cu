// r128.cu — the EBUr128 plugin's audio cycle for N instances of 1..5 channels (stereo: the plugin itself), and of 1..32 channels
// with caller-given channel weights (b200m_r128_create_weighted): EBU R128 loudness + optional dBTP.
//
// Mirrors what ebur128_run does between its atom parsing and atom forging (src/ebulv2.cc:341-367), with nchan channels in
// Ebu_r128_proc's order L R C Ls Rs:
//   ebu->process (n, {in0 .. in[nchan-1]});  if (dbtp_enable) mtr[c]->process_max (in[c]) for every c;
//   lm/mm/ls/ms/il/rn/rx getters;  t = mtr[0]->read (); t = t > mtr[c]->read () ? t : mtr[c]->read () for c >= 1;
//   tp = coef_to_db (t);  tp_max = max (tp_max, tp)
// It composes the EBU bank (ebu.cu) and the true-peak bank (tpk.cu) over ONE host->device copy of the block.
#include <math.h>
#include <stdlib.h>
#include <vector>
#include "common.cuh"
#include "ebu_kw.cuh"

namespace b200m {

// coef_to_db (src/ebulv2.cc:227-230) and the tp_max hold (:360-367) run in the epilogue of the true-peak kernels (tpk.cu) when an
// instance's channels never leave an 8-channel true-peak group (1, 2, 4 channels).  With 3 or 5 they leave every channel's read()
// in lin[] (R128Hold) and this kernel, one thread per instance behind them, folds the instance's reads in channel order.
// rlen (a ragged block): an instance with length 0 did not run, its hold stays.
template <int NCHAN>
__global__ void r128_hold_kernel (int n_inst, const float* __restrict__ lin, float* __restrict__ tpmax, const uint32_t* __restrict__ rlen)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_inst || (rlen && rlen[i] == 0)) return;
    float t = lin[(size_t)i * NCHAN];
#pragma unroll
    for (int c = 1; c < NCHAN; ++c) { const float v = lin[(size_t)i * NCHAN + c]; t = t > v ? t : v; }
    r128_hold (tpmax + i, t);
}
// the same fold for a weighted bank: nch = 1..32 channels per instance, known at run time
__global__ void r128_hold_kernel_w (int n_inst, int nch, const float* __restrict__ lin, float* __restrict__ tpmax, const uint32_t* __restrict__ rlen)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_inst || (rlen && rlen[i] == 0)) return;
    float t = lin[(size_t)i * nch];
    for (int c = 1; c < nch; ++c) { const float v = lin[(size_t)i * nch + c]; t = t > v ? t : v; }
    r128_hold (tpmax + i, t);
}
__global__ void r128_fill_kernel (int n, float* p, float v) { const int i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = v; }
// the same for the instances of a ragged block that ran (rlen[i] > 0)
__global__ void r128_fill_ran_kernel (int n, float* p, float v, const uint32_t* __restrict__ rlen)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && rlen[i] != 0) p[i] = v;
}

// Per-instance dBTP.  An instance with dBTP off runs no process_max (src/ebulv2.cc:344-347): its nchan TruePeakdsp histories
// stay frozen and its hold is -inf after the cycle (:365-366).  In a cycle with a mixed mask the true-peak kernels process every
// channel; behind them r128_dbtp_fix_kernel puts the frozen histories (stash) back into the history the next block reads and
// clears the hold of the disabled instances (in a ragged block: of those that ran; a disabled instance's histories stay frozen whatever
// its length).  One thread per (instance, history float); nh = nchan x 48 history floats per instance.
__global__ void r128_dbtp_stash_kernel (int n_inst, int nh, const uint8_t* __restrict__ off, const float* __restrict__ hist, float* __restrict__ stash)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_inst * nh || !off[t / nh]) return;
    stash[t] = hist[t];                           // the channels of instance i are nchan i .. nchan i + nchan - 1: its floats are contiguous
}
__global__ void r128_dbtp_fix_kernel (int n_inst, int nh, const uint8_t* __restrict__ off, const float* __restrict__ stash, float* __restrict__ hist,
                                      float* __restrict__ tpmax, const uint32_t* __restrict__ rlen)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_inst * nh) return;
    const int i = t / nh;
    if (!off[i]) return;
    hist[t] = stash[t];
    if (t % nh == 0 && !(rlen && rlen[i] == 0)) tpmax[i] = -INFINITY;
}

}  // namespace b200m

// sliced process entry point of the true-peak bank and the fused K-weighting + true-peak kernel (tpk.cu); the EBU bank's: ebu_kw.cuh
int tpk_process_sliced (b200m_tpk* h, const float* d_in, size_t stride, uint32_t nfram, uint32_t tp_mode, cudaStream_t st, int nsl, const uint32_t* bounds, cudaEvent_t* ready,
                        b200m::R128Hold r128, bool pdl, const void* dr, const uint32_t* rlen);
bool tpk_r128_fused_ok (const b200m_tpk* h, const float* d_in, size_t stride, uint32_t nfram);
float* tpk_hist (b200m_tpk* h);
int tpk_r128_fused (b200m_tpk* h, const b200m::EbuK1Args& a, float* r128_tpmax, cudaStream_t st);

using namespace b200m;

constexpr int R128_SLICES = 8;        // maximum; default 4 (B200M_R128_SLICES)

struct b200m_r128 {
    int device; uint32_t n_inst, nchan;
    bool weighted = false;               // b200m_r128_create_weighted with other than the default weights (1..32 channels)
    int dbtp;                            // some instance has dBTP on: the true-peak kernels run
    // per-instance dBTP switch (host), its device copy (uploaded before the first mixed cycle after a change) and the frozen
    // histories of the disabled instances; stash_ok: the stash holds every disabled instance's current frozen history
    std::vector<uint8_t> off; uint32_t n_off = 0; bool off_dirty = true, stash_ok = false, fixed = false;
    uint8_t* d_off = nullptr; float* d_stash = nullptr;
    b200m_ebu* ebu = nullptr; b200m_tpk* tpk = nullptr;
    float* d_tpmax = nullptr;
    float* d_tplin = nullptr;            // 3 or 5 channels, weighted banks: every channel's read() of the cycle, folded by r128_hold_kernel
    R128Hold hold () const { return {d_tpmax, d_tplin, (int)nchan}; }
    // own: EBU kernels + joins (host path);  side: true-peak kernels (run concurrently with the latency-bound EBU
    // kernel);  copy: host->device slices, so that the copy of slice s+1 overlaps the kernels of slice s
    cudaStream_t own = nullptr, side = nullptr, copy = nullptr;
    cudaEvent_t ev_tp = nullptr, ev_done = nullptr, ev_pre = nullptr, ev_ready[R128_SLICES] = {nullptr};
    HostStage stage; bool last_host = false; int concurrent = 1, slices = R128_SLICES;
};

static int env_int (const char* name, int dflt) { const char* v = getenv (name); return v ? atoi (v) : dflt; }

struct R128Step { b200m_r128* h; const float* d_in; size_t stride; uint32_t nfram; cudaStream_t st; const uint32_t* bc; const uint32_t* d_len; };

// device path: the true-peak kernel goes onto the caller's stream right behind the first K-weighting launch, with
// programmatic dependent launch, so that the two kernels share the SMs (see r128_run)
static int r128_tp_behind_k1 (void* p)
{
    R128Step* a = (R128Step*)p;
    return tpk_process_sliced (a->h->tpk, a->d_in, a->stride, a->nfram, B200M_TP_MODE_MAX, a->st, 1, a->bc, nullptr, a->h->hold (), true, nullptr, a->d_len);
}

// device path, fused: one kernel does K1's work and the true-peak maximum over one shared-memory copy of the block (tpk.cu)
static int r128_fused_k1 (void* p, const EbuK1Args& a)
{
    R128Step* s = (R128Step*)p;
    return tpk_r128_fused (s->h->tpk, a, s->h->d_tpmax, s->st);
}

// len (host, every entry <= nfram, some != nfram): a ragged block, instance i runs its cycle over its first len[i] frames; nullptr: all nfram
static int r128_run (b200m_r128* h, const float* d_in, size_t stride, uint32_t nfram, cudaStream_t st, int nsl, cudaEvent_t* ready,
                     const uint32_t* len = nullptr)
{
    uint32_t bi[R128_SLICES + 1], bc[R128_SLICES + 1];
    for (int s = 0; s <= nsl; ++s) { bi[s] = (uint32_t)((uint64_t)h->n_inst * s / nsl); bc[s] = h->nchan * bi[s]; }
    // The K-weighting kernel is latency bound on 4 warps per SM and the true-peak kernel issue bound: run together they
    // cost little more than the true-peak kernel alone, PROVIDED the K-weighting CTAs are resident first (104 KB of shared
    // memory each: they do not fit once the true-peak CTAs fill an SM).
    //  * device path (B200M_R128_CONCURRENT >= 2): same stream; the K-weighting kernel triggers programmatic launch
    //    completion at its start and the true-peak kernel is launched behind it with the programmatic-serialization
    //    attribute -> deterministic order, no events.  The true-peak kernel's epilogue does read() x nchan + coef_to_db + the
    //    tp_max hold per instance (3, 5 channels: r128_hold_kernel behind it) and ends with griddepcontrol.wait, so everything
    //    queued behind it is ordered after both.
    //  * sliced host path (>= 1): true-peak kernels on the side stream, each slice behind its copy event.
    // B200M_R128_CONCURRENT=0 serialises everything on one stream.
    // Tolerance mode on the device path runs neither: one fused kernel takes K1's place (r128_fused_kernel, tpk.cu) when the
    // true-peak bank would take the tensor-core path, the block is 16-byte aligned with nfram % 4 == 0, its chunk list fits one K1
    // launch and the bank is large enough to fill the GPU with 128-channel (3 and 5 channels: 120-channel) slabs.
    // 3 and 5 channels outside the fused kernel: r128_hold_kernel behind the true-peak kernels folds the hold.
    // A ragged block: one upload of the lengths, read by the K-weighting, fragment and true-peak kernels.  The true-peak FIR is
    // tpmax_kernel in both precision modes (tpk_process_sliced): no fused kernel.
    const uint32_t* d_len = nullptr;
    if (len && !(d_len = ebu_upload_len (h->ebu, len, st))) return B200M_E_CUDA;
    const bool mixed = h->n_off && h->n_off < h->n_inst;
    if (mixed) {
        // the first mixed cycle after a change: device mask, then the frozen histories of the disabled instances.  Until now every
        // disabled instance's history has stayed in the buffer the next block reads (fixed up after mixed cycles, untouched by
        // cycles without the true-peak kernels), so that is where the stash is taken from.
        const int nh = (int)h->nchan * 48, nt = (int)h->n_inst * nh;
        if (h->off_dirty) { B200M_CUDA (cudaMemcpyAsync (h->d_off, h->off.data (), h->n_inst, cudaMemcpyHostToDevice, st)); h->off_dirty = false; }
        if (!h->stash_ok) {
            r128_dbtp_stash_kernel<<<(nt + 255) / 256, 256, 0, st>>> ((int)h->n_inst, nh, h->d_off, tpk_hist (h->tpk), h->d_stash);
            B200M_LAUNCHED (1);
            h->stash_ok = true;
        }
    }
    // weighted banks have no fused form: they keep the two-kernel cycle (K1 + the true-peak kernel behind it), see DESIGN.md §3
    const bool fused = !ready && !d_len && h->dbtp && !h->weighted && tpk_r128_fused_ok (h->tpk, d_in, stride, nfram) && ebu_single_k1 (h->ebu, nfram);
    const bool pdl = !fused && h->dbtp && h->concurrent >= 2 && !ready;
    const bool conc = h->dbtp && h->concurrent >= 1 && ready;
    // the side stream's true-peak kernels read the history that the stash / fix-up kernels on st touch
    if (conc && (mixed || h->fixed || d_len)) { B200M_CUDA (cudaEventRecord (h->ev_pre, st)); B200M_CUDA (cudaStreamWaitEvent (h->side, h->ev_pre, 0)); }
    h->fixed = mixed && h->dbtp;
    R128Step step = {h, d_in, stride, nfram, st, bc, d_len};
    if (int rc = ebu_process_sliced (h->ebu, d_in, stride, nfram, st, nsl, bi, ready, pdl ? r128_tp_behind_k1 : nullptr, &step,
                                     fused ? r128_fused_k1 : nullptr, len, d_len)) return rc;
    if (h->dbtp) {
        if (!pdl && !fused) {
            if (int rc = tpk_process_sliced (h->tpk, d_in, stride, nfram, B200M_TP_MODE_MAX, conc ? h->side : st, nsl, bc, conc ? ready : nullptr, h->hold (), false, nullptr, d_len)) return rc;
            if (conc) { B200M_CUDA (cudaEventRecord (h->ev_tp, h->side)); B200M_CUDA (cudaStreamWaitEvent (st, h->ev_tp, 0)); }
        }
        if (h->d_tplin && !fused) {                        // behind every slice's true-peak kernel, before the fix-up clears holds
            const int nb = (h->n_inst + 255) / 256;
            if (h->weighted) r128_hold_kernel_w<<<nb, 256, 0, st>>> ((int)h->n_inst, (int)h->nchan, h->d_tplin, h->d_tpmax, d_len);
            else if (h->nchan == 3) r128_hold_kernel<3><<<nb, 256, 0, st>>> ((int)h->n_inst, h->d_tplin, h->d_tpmax, d_len);
            else r128_hold_kernel<5><<<nb, 256, 0, st>>> ((int)h->n_inst, h->d_tplin, h->d_tpmax, d_len);
            B200M_LAUNCHED (1);
        }
        if (mixed) {                                       // behind the true-peak kernels on st, and behind the history swap on the host
            const int nh = (int)h->nchan * 48, nt = (int)h->n_inst * nh;
            r128_dbtp_fix_kernel<<<(nt + 255) / 256, 256, 0, st>>> ((int)h->n_inst, nh, h->d_off, h->d_stash, tpk_hist (h->tpk), h->d_tpmax, d_len);
            B200M_LAUNCHED (1);
        }
    } else {
        if (d_len) r128_fill_ran_kernel<<<(h->n_inst + 255) / 256, 256, 0, st>>> ((int)h->n_inst, h->d_tpmax, -INFINITY, d_len);
        else r128_fill_kernel<<<(h->n_inst + 255) / 256, 256, 0, st>>> ((int)h->n_inst, h->d_tpmax, -INFINITY);   // :365-366
        B200M_LAUNCHED (1);
    }
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

static void r128_set_dbtp (b200m_r128* h, int32_t inst, bool on)
{
    const uint32_t a = inst < 0 ? 0 : (uint32_t)inst, e = inst < 0 ? h->n_inst : (uint32_t)inst + 1;
    for (uint32_t i = a; i < e; ++i) {
        if (h->off[i] == (uint8_t)!on) continue;
        h->off[i] = (uint8_t)!on; h->n_off += on ? -1 : 1; h->off_dirty = true;
        if (!on) h->stash_ok = false;                      // a newly frozen history is not in the stash yet
    }
    h->dbtp = h->n_off < h->n_inst;
}

extern "C" {

int b200m_r128_create (b200m_r128** out, int device, uint32_t n_inst, float fsamp, int dbtp_enable)
{
    return b200m_r128_create_nch (out, device, n_inst, 2, fsamp, dbtp_enable);
}

}  // extern "C"

// gains == nullptr: the default weights of a 1..5-channel bank; otherwise a weighted bank (validated by the caller)
static int r128_create (b200m_r128** out, int device, uint32_t n_inst, uint32_t nchan, const float* gains, float fsamp, int dbtp_enable)
{
    b200m_r128* h = new (std::nothrow) b200m_r128;
    if (!h) return set_err (B200M_E_NOMEM, "host allocation failed");
    h->device = device; h->n_inst = n_inst; h->nchan = nchan; h->weighted = gains != nullptr;
    h->off.assign (n_inst, 0); h->n_off = 0;
    r128_set_dbtp (h, -1, dbtp_enable != 0);
    h->concurrent = env_int ("B200M_R128_CONCURRENT", 2);      // 0: serial, 1: sliced host path only, 2: device path too
    h->slices = env_int ("B200M_R128_SLICES", 4);
    if (h->slices < 1) h->slices = 1;
    if (h->slices > R128_SLICES) h->slices = R128_SLICES;
    int rc = gains ? b200m_ebu_create_weighted (&h->ebu, device, n_inst, nchan, gains, fsamp)
                   : b200m_ebu_create (&h->ebu, device, n_inst, nchan, fsamp);                // ebu->init (nchan, rate), src/ebulv2.cc:190
    if (!rc) rc = b200m_tpk_create (&h->tpk, device, nchan * n_inst, fsamp, B200M_TPK_TRUEPEAK);   // nchan x TruePeakdsp, :192-196
    if (!rc) {
        DeviceGuard g (device);
        cudaError_t e = cudaMalloc ((void**)&h->d_tpmax, n_inst * sizeof (float));
        if (e == cudaSuccess) e = cudaMalloc ((void**)&h->d_off, n_inst);
        if (e == cudaSuccess) e = cudaMalloc ((void**)&h->d_stash, (size_t)n_inst * nchan * 48 * sizeof (float));
        if (e == cudaSuccess && (nchan == 3 || nchan == 5 || gains)) e = cudaMalloc ((void**)&h->d_tplin, (size_t)n_inst * nchan * sizeof (float));
        for (cudaStream_t* sp : {&h->own, &h->side, &h->copy}) if (e == cudaSuccess) e = cudaStreamCreateWithFlags (sp, cudaStreamNonBlocking);
        for (cudaEvent_t* ep : {&h->ev_tp, &h->ev_done, &h->ev_pre}) if (e == cudaSuccess) e = cudaEventCreateWithFlags (ep, cudaEventDisableTiming);
        for (int s = 0; s < R128_SLICES; ++s) if (e == cudaSuccess) e = cudaEventCreateWithFlags (&h->ev_ready[s], cudaEventDisableTiming);
        if (e == cudaSuccess) {
            r128_fill_kernel<<<(n_inst + 255) / 256, 256>>> ((int)n_inst, h->d_tpmax, -INFINITY);
            B200M_LAUNCHED (1);
            e = cudaDeviceSynchronize ();
        }
        if (e != cudaSuccess) rc = cuda_fail (e, "r128_create", __FILE__, __LINE__);
    }
    if (rc) { b200m_r128_destroy (h); return rc; }
    *out = h;
    return 0;
}

extern "C" {

int b200m_r128_create_nch (b200m_r128** out, int device, uint32_t n_inst, uint32_t nchan, float fsamp, int dbtp_enable)
{
    if (!out) return set_err (B200M_E_INVAL, "NULL out pointer");
    *out = nullptr;
    if (nchan < 1 || nchan > 5) return set_err (B200M_E_INVAL, "nchan %u outside 1..5", nchan);
    return r128_create (out, device, n_inst, nchan, nullptr, fsamp, dbtp_enable);
}

int b200m_r128_create_weighted (b200m_r128** out, int device, uint32_t n_inst, uint32_t nchan, const float* gains, float fsamp, int dbtp_enable)
{
    if (!out) return set_err (B200M_E_INVAL, "NULL out pointer");
    *out = nullptr;
    if (int rc = ebu_check_gains (nchan, gains)) return rc;
    // the reference's own weights for its channel count: exactly the bank b200m_r128_create_nch makes
    return r128_create (out, device, n_inst, nchan, ebu_default_gains (nchan, gains) ? nullptr : gains, fsamp, dbtp_enable);
}

int b200m_r128_destroy (b200m_r128* h)
{
    if (!h) return 0;
    b200m_ebu_destroy (h->ebu); b200m_tpk_destroy (h->tpk);
    DeviceGuard g (h->device);
    cudaDeviceSynchronize ();
    cudaFree (h->d_tpmax); cudaFree (h->d_off); cudaFree (h->d_stash); cudaFree (h->d_tplin); h->stage.release ();
    for (cudaStream_t sp : {h->own, h->side, h->copy}) if (sp) cudaStreamDestroy (sp);
    for (cudaEvent_t ep : {h->ev_tp, h->ev_done, h->ev_pre}) if (ep) cudaEventDestroy (ep);
    for (int s = 0; s < R128_SLICES; ++s) if (h->ev_ready[s]) cudaEventDestroy (h->ev_ready[s]);
    delete h;
    return 0;
}

int b200m_r128_control (b200m_r128* h, int32_t inst, int cmd, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    void* st = h->last_host ? (void*)h->own : stream;
    switch (cmd) {
    case B200M_R128_START: return b200m_ebu_integr_start (h->ebu, inst, st);
    case B200M_R128_PAUSE: return b200m_ebu_integr_pause (h->ebu, inst, st);
    case B200M_R128_RESET:                                  // ebu_reset (src/ebulv2.cc:45-61): integr_reset + tp_max = -inf
    case B200M_R128_CLEAR_TPMAX: {                          // tp_max = -inf alone: what a cycle with dBTP disabled leaves behind (:365-366)
        if (inst >= (int32_t)h->n_inst) return set_err (B200M_E_INVAL, "bad instance %d", inst);
        DeviceGuard g (h->device);
        const int first = inst < 0 ? 0 : inst, cnt = inst < 0 ? (int)h->n_inst : 1;
        r128_fill_kernel<<<(cnt + 255) / 256, 256, 0, (cudaStream_t)st>>> (cnt, h->d_tpmax + first, -INFINITY);
        B200M_LAUNCHED (1);
        B200M_CUDA (cudaGetLastError ());
        return cmd == B200M_R128_RESET ? b200m_ebu_integr_reset (h->ebu, inst, st) : 0;
    }
    case B200M_R128_CLEAR:                                  // a fresh instance in this slot (shared banks: a plugin left, another may join)
    case B200M_R128_NEW: {                                  // ... whose 50 ms fragment clock starts with the next block
        if (inst < 0 || inst >= (int32_t)h->n_inst) return set_err (B200M_E_INVAL, "bad instance %d", inst);
        DeviceGuard g (h->device);
        r128_fill_kernel<<<1, 32, 0, (cudaStream_t)st>>> (1, h->d_tpmax + inst, -INFINITY);
        B200M_LAUNCHED (1);
        B200M_CUDA (cudaGetLastError ());
        if (int rc = cmd == B200M_R128_NEW ? b200m_ebu_reset (h->ebu, inst, st) : b200m_ebu_clear (h->ebu, inst, st)) return rc;
        if (h->off[inst]) h->stash_ok = false;             // its frozen histories are now the cleared ones
        for (uint32_t c = 0; c < h->nchan; ++c)
            if (int rc = b200m_tpk_clear (h->tpk, (int32_t)(h->nchan * inst + c), st)) return rc;
        return 0;
    }
    default: return set_err (B200M_E_INVAL, "unknown control %d", cmd);
    }
}

int b200m_r128_run_device (b200m_r128* h, const float* d_in, size_t stride, uint32_t nfram, void* stream)
{
    if (int rc = check_block_args (h, d_in, stride, nfram)) return rc;
    DeviceGuard g (h->device);
    h->last_host = false;
    return r128_run (h, d_in, stride, nfram, (cudaStream_t)stream, 1, nullptr);
}

int b200m_r128_run_ragged_device (b200m_r128* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream)
{
    if (int rc = check_block_args (h, d_in, stride, nfram)) return rc;
    const int rag = ebu_ragged_check (h->ebu, nfram, len);
    if (rag < 0) return rag;
    if (!rag) return b200m_r128_run_device (h, d_in, stride, nfram, stream);        // every length is nfram: the plain call
    DeviceGuard g (h->device);
    h->last_host = false;
    return r128_run (h, d_in, stride, nfram, (cudaStream_t)stream, 1, nullptr, len);
}

static int r128_run_host (b200m_r128* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len);

int b200m_r128_run_host (b200m_r128* h, const float* in, size_t stride, uint32_t nfram)
{
    return r128_run_host (h, in, stride, nfram, nullptr);
}

int b200m_r128_run_ragged_host (b200m_r128* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len)
{
    if (int rc = check_block_args (h, in, stride, nfram)) return rc;
    const int rag = ebu_ragged_check (h->ebu, nfram, len);
    if (rag < 0) return rag;
    return r128_run_host (h, in, stride, nfram, rag ? len : nullptr);
}

}  // extern "C"

static int r128_run_host (b200m_r128* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len)
{
    if (int rc = check_block_args (h, in, stride, nfram)) return rc;
    DeviceGuard g (h->device);
    B200M_ENTER_HOST_PATH (h);
    const size_t nch = (size_t)h->nchan * h->n_inst;
    if (h->stage.ensure (nch, nfram)) return set_err (B200M_E_NOMEM, "staging buffer allocation failed");
    // the staging buffer is single: the next copy may only start when the previous cycle's kernels have read it
    if (h->last_host) B200M_CUDA (cudaStreamWaitEvent (h->copy, h->ev_done, 0));
    const int nsl = h->n_inst >= 64 ? h->slices : 1;
    for (int s = 0; s < nsl; ++s) {
        const size_t r0 = h->nchan * ((uint64_t)h->n_inst * s / nsl), r1 = h->nchan * ((uint64_t)h->n_inst * (s + 1) / nsl);
        if (stride == nfram && h->stage.cap == nfram)          // both sides dense: one contiguous DMA per slice (faster than 4 KB rows)
            B200M_CUDA (cudaMemcpyAsync (h->stage.d + r0 * h->stage.cap, in + r0 * stride, (r1 - r0) * (size_t)nfram * sizeof (float), cudaMemcpyHostToDevice, h->copy));
        else
            B200M_CUDA (cudaMemcpy2DAsync (h->stage.d + r0 * h->stage.cap, h->stage.cap * sizeof (float), in + r0 * stride, stride * sizeof (float),
                                           (size_t)nfram * sizeof (float), r1 - r0, cudaMemcpyHostToDevice, h->copy));
        B200M_CUDA (cudaEventRecord (h->ev_ready[s], h->copy));
    }
    h->last_host = true;
    if (int rc = r128_run (h, h->stage.d, h->stage.cap, nfram, h->own, nsl, h->ev_ready, len)) return rc;
    B200M_CUDA (cudaEventRecord (h->ev_done, h->own));
    return 0;
}

extern "C" {

int b200m_r128_results (b200m_r128* h, b200m_ebu_result* ebu_out, float* tp_max_db, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    DeviceGuard g (h->device);
    cudaStream_t st = h->last_host ? h->own : (cudaStream_t)stream;
    if (tp_max_db) B200M_CUDA (cudaMemcpyAsync (tp_max_db, h->d_tpmax, h->n_inst * sizeof (float), cudaMemcpyDeviceToHost, st));
    if (ebu_out) return b200m_ebu_results (h->ebu, ebu_out, st);
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_r128_set_dbtp (b200m_r128* h, int enable) { return b200m_r128_set_dbtp_inst (h, -1, enable); }

int b200m_r128_set_dbtp_inst (b200m_r128* h, int32_t inst, int enable)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    if (inst < -1 || inst >= (int32_t)h->n_inst) return set_err (B200M_E_INVAL, "bad instance %d", inst);
    r128_set_dbtp (h, inst, enable != 0);                  // takes effect with the next run: self->dbtp_enable (src/ebulv2.cc:316-317,344-347)
    return 0;
}

int b200m_r128_set_precision (b200m_r128* h, int mode)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    return b200m_tpk_set_precision (h->tpk, mode);         // the EBU R128 part is always exact: it feeds the integer histograms
}

int b200m_r128_histogram (b200m_r128* h, uint32_t inst, int32_t* hist_M, int32_t* hist_S, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    return b200m_ebu_histogram (h->ebu, inst, hist_M, hist_S, h->last_host ? (void*)h->own : stream);
}

// snapshot = [u64 ebu bytes][u64 tpk bytes][ebu blob][tpk blob][tp_max floats][16 bytes of flags][per-instance dBTP off bytes].
// The frozen histories are in the tpk blob (the history the next block reads), so the stash is retaken after a restore.  The ebu
// blob's header records nchan: a blob of a bank with another channel count has other sizes (or that header) and is refused.
size_t b200m_r128_snapshot_size (b200m_r128* h)
{
    if (!h) return 0;
    return 16 + b200m_ebu_snapshot_size (h->ebu) + b200m_tpk_snapshot_size (h->tpk) + (((size_t)h->n_inst * 4 + 15) & ~size_t (15)) + 16
        + (((size_t)h->n_inst + 15) & ~size_t (15));
}

int b200m_r128_snapshot (b200m_r128* h, void* buf, size_t bytes, void* stream)
{
    if (!h || !buf || bytes < b200m_r128_snapshot_size (h)) return set_err (B200M_E_INVAL, "bad argument / buffer too small");
    DeviceGuard g (h->device);
    void* st = h->last_host ? (void*)h->own : stream;
    const uint64_t eb = b200m_ebu_snapshot_size (h->ebu), tb = b200m_tpk_snapshot_size (h->tpk);
    uint8_t* o = (uint8_t*)buf;
    memcpy (o, &eb, 8); memcpy (o + 8, &tb, 8); o += 16;
    if (int rc = b200m_ebu_snapshot (h->ebu, o, eb, st)) return rc;
    o += eb;
    if (int rc = b200m_tpk_snapshot (h->tpk, o, tb, st)) return rc;
    o += tb;
    B200M_CUDA (cudaMemcpyAsync (o, h->d_tpmax, (size_t)h->n_inst * 4, cudaMemcpyDeviceToHost, (cudaStream_t)st));
    B200M_CUDA (cudaStreamSynchronize ((cudaStream_t)st));
    o += ((size_t)h->n_inst * 4 + 15) & ~size_t (15);
    const int32_t fl[4] = {h->dbtp, 0, 0, 0};
    memcpy (o, fl, 16);
    memcpy (o + 16, h->off.data (), h->n_inst);
    return 0;
}

int b200m_r128_restore (b200m_r128* h, const void* buf, size_t bytes, void* stream)
{
    if (!h || !buf || bytes < b200m_r128_snapshot_size (h)) return set_err (B200M_E_INVAL, "bad argument / buffer too small");
    DeviceGuard g (h->device);
    void* st = h->last_host ? (void*)h->own : stream;
    uint64_t eb, tb;
    const uint8_t* o = (const uint8_t*)buf;
    memcpy (&eb, o, 8); memcpy (&tb, o + 8, 8); o += 16;
    if (eb != b200m_ebu_snapshot_size (h->ebu) || tb != b200m_tpk_snapshot_size (h->tpk)) return set_err (B200M_E_INVAL, "snapshot does not match this bank");
    if (int rc = b200m_ebu_restore (h->ebu, o, eb, st)) return rc;
    o += eb;
    if (int rc = b200m_tpk_restore (h->tpk, o, tb, st)) return rc;
    o += tb;
    B200M_CUDA (cudaMemcpyAsync (h->d_tpmax, o, (size_t)h->n_inst * 4, cudaMemcpyHostToDevice, (cudaStream_t)st));
    B200M_CUDA (cudaStreamSynchronize ((cudaStream_t)st));
    o += ((size_t)h->n_inst * 4 + 15) & ~size_t (15);
    memcpy (h->off.data (), o + 16, h->n_inst);
    h->n_off = 0;
    for (uint8_t v : h->off) h->n_off += v ? 1 : 0;
    h->dbtp = h->n_off < h->n_inst;
    h->off_dirty = true; h->stash_ok = false;
    return 0;
}

b200m_ebu* b200m_r128_ebu (b200m_r128* h) { return h ? h->ebu : nullptr; }
b200m_tpk* b200m_r128_tpk (b200m_r128* h) { return h ? h->tpk : nullptr; }

}  // extern "C"
