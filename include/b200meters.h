/* b200meters.h — C ABI of the CUDA batched audio-metering engine (H100, sm_90a).
 *
 * One "bank" = N independent instances of one reference DSP class, all processed by one CUDA
 * kernel launch per process() call.  Entry points mirror, one for one, the methods an LV2 host
 * reaches through x42/meters.lv2's run() callbacks; each declaration cites the reference
 * interface it replaces (paths relative to the reference tree).
 *
 * Conventions
 *  - plain C, no CUDA/torch types: device pointers and streams travel as void*.
 *  - every function returns 0 on success or a negative B200M_E_* code; nothing throws.
 *  - audio is planar float32, exactly what an LV2 host connects to an audio port
 *    (src/meters.cc:257-296): channel k (k = inst*nchan + c) of a process call starts at
 *    in + k*stride and holds nfram samples (interleaved integer PCM converts to it on the device:
 *    b200m_pcm_planar_device).  `*_process_device` takes a device pointer and is
 *    asynchronous on `stream` (a cudaStream_t, NULL = legacy default stream);
 *    `*_process_host` takes a host pointer (pinned memory recommended: b200m_host_alloc),
 *    performs the host->device copy itself and is asynchronous on the bank's own stream.
 *  - a bank may switch path between any two calls and the library keeps program order: the
 *    first host-path call after device-path calls synchronises the device, the first
 *    device-path call after host-path calls waits for the bank's own stream.  Consecutive
 *    device-path calls on different streams must be ordered by the caller.
 *  - getters, controls and `*_read_device` run on the bank's own stream after a host-path call
 *    and on the stream they are given after a device-path call: pass the stream of the last
 *    device-path call.  A correlation bank attached to a phasewheel bank (b200m_pw_attach_cor)
 *    follows the phasewheel bank: after its host-path call the correlation bank is read as after
 *    one of its own.
 *  - `*_read_device` mirrors the reference's read()/getter step on the device (including its
 *    reset-latch side effects) and stores the values in a device result block;
 *    `*_results` copies that block to the host (synchronises the stream it was given).
 *  - there is NO CPU fallback: a bank cannot be created without a CUDA device, and every
 *    sample is processed by the sm_90a kernels in meters.lv2_b200/csrc/.
 */
#ifndef B200METERS_H
#define B200METERS_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)   /* the library is built with -fvisibility=hidden */
#endif

#define B200M_ABI_VERSION 1

enum {
    B200M_OK            =  0,
    B200M_E_INVAL       = -1,   /* bad argument (NULL handle, n out of range, bad stride ...) */
    B200M_E_NOMEM       = -2,   /* host or device allocation failed */
    B200M_E_CUDA        = -3,   /* CUDA runtime error: see b200m_last_error() */
    B200M_E_UNSUPPORTED = -4,   /* valid in the reference, not provided by this engine */
    B200M_E_NODEVICE    = -5    /* no CUDA device: the engine has no CPU path */
};

#define B200M_MAX_BLOCK 8192u     /* TruePeakdsp::process asserts n <= 8192 (jmeters/truepeakdsp.cc:43-44);
                                     robtk/jackwrap.c:35 MAXPERIOD 8192 */
#define B200M_HIST_LEN  751       /* Ebu_r128_hist bins, -70.0 .. +5.0 dB (ebumeter/ebu_r128_proc.cc:34) */

int         b200m_abi_version (void);
const char* b200m_last_error (void);            /* thread-local text of the last failure */
int         b200m_device_count (void);
/* pinned host memory for process_host()/results(): cudaHostAlloc / cudaFreeHost */
int         b200m_host_alloc (void** p, size_t bytes);
int         b200m_host_free (void* p);
/* number of kernel launches issued by this library since load (bench.py's gpu_launches) */
uint64_t    b200m_launch_count (void);

/* ALU ceilings measured on the device:
 * kind 0 = fp32 unfused FMUL+FADD issue rate, kind 1 = fp64 DMUL+DADD;
 * result in 1e9 lane-operations/s. */
int         b200m_peak_probe (int device, int kind, double* gops);

/* Self-test hook: log10f of the `count` floats whose bit patterns are first_bits, first_bits + 1, ... written to the DEVICE
 * array d_out, evaluated by the device function every loudness / dB value of the engine goes through (a restatement of
 * glibc's log10f: the reference bins log10f results into integer histograms, ebumeter/ebu_r128_proc.cc:66-79,116-141,259).
 * tests/test_log10f_sweep_gpu.py sweeps all 2^31 non-negative floats against the host libm with it. */
int         b200m_selftest_log10f (int device, uint32_t first_bits, uint32_t count, float* d_out, void* stream);

/* Host-side coefficient design, callable without a GPU (pure functions of the sample rate, computed with
 * the host libm in the reference's expression types so that every value is bitwise the reference's):
 *   ebu : detect_init (ebumeter/ebu_r128_proc.cc:263-293)           -> a0 a1 a2 b1 b2 c3 c4
 *   tpk : TruePeakdsp::init (jmeters/truepeakdsp.cc:148-157), zita table (zita-resampler/resampler-table.cc:
 *         52-75; hl=24 np=4 fr=1), Kmeterdsp::init (jmeters/kmeterdsp.cc:47-54) -> w1 w2 w3 g | ctab | omega hold
 *   cor : Stcorrdsp::init (jmeters/stcorrdsp.cc:85-93)              -> w1 w2
 *   spec: spectrum_instantiate band table + bandpass_setup (src/spectrumlv2.c:100-118, src/spectr.c:89-206)
 *         -> W[30][6][6] = a0 a1 a2 b0 b1 b2 per section */
int b200m_design_ebu (float fsamp, float out7[7]);
int b200m_design_tpk (float fsamp, float w[4], float ctab[120], float km[2]);
int b200m_design_cor (int fsamp, float flp, float tcf, float w[2]);
int b200m_design_spec (double rate, double* W1080);

/* ======================================================================================
 * EBU R128 loudness bank — replaces LV2M::Ebu_r128_proc (ebumeter/ebu_r128_proc.h:66-125)
 * as driven by ebur128_run (src/ebulv2.cc:341-358).
 * ====================================================================================== */
typedef struct b200m_ebu b200m_ebu;

typedef struct b200m_ebu_result {          /* getters, ebumeter/ebu_r128_proc.h:81-89 */
    float loudness_M, maxloudn_M, loudness_S, maxloudn_S;
    float integrated, integ_thr, range_min, range_max, range_thr;
    int32_t hist_M_count, hist_S_count;    /* :93-94 */
    float   frag_power;                    /* last completed 50 ms fragment power (_power[_wrind-1]) */
} b200m_ebu_result;

/* Ebu_r128_proc() + init(nchan, fsamp) (:166-173) for n_inst instances.  nchan 1..5 (the EBUr128 plugin uses 2, src/ebulv2.cc:190;
 * 3..5: surround layouts with the channel gains 1 1 1 1.41 1.41 of ebu_r128_proc.cc:29). */
int b200m_ebu_create (b200m_ebu** out, int device, uint32_t n_inst, uint32_t nchan, float fsamp);
/* The same bank with nchan = 1..32 channels per instance and caller-given channel weights: the per-chunk channel sum is
 * si = gains[0] * sj0, then si += gains[c] * sj_c in channel order, in fp32 (detect_process, ebu_r128_proc.cc:328-330, with these
 * weights; mono {2.0f} is the reference's 2 * sj).  Gains must be finite and >= 0 with at least one > 0, else B200M_E_INVAL and
 * *out = NULL.  The reference's own weights for 1..5 channels (mono {2}, else 1 1 1 1.41 1.41) give exactly b200m_ebu_create's bank;
 * any other set runs the run-time channel-count K-weighting kernel.  Snapshots of a weighted bank record nchan and the gains and
 * restore only into a bank with the same ones (bitwise). */
int b200m_ebu_create_weighted (b200m_ebu** out, int device, uint32_t n_inst, uint32_t nchan, const float* gains, float fsamp);
/* ITU-R BS.1770-4 channel weights from loudspeaker positions in degrees: 1.41 when |elevation| < 30 and 60 <= |azimuth| <= 120
 * (azimuth taken modulo 360 into -180 .. 180), 1.0 otherwise.  Host only: needs no device.  Non-finite positions: B200M_E_INVAL. */
int b200m_bs1770_weights (uint32_t n, const float* azimuth_deg, const float* elevation_deg, float* gains);
int b200m_ebu_destroy (b200m_ebu* h);
/* Ebu_r128_proc::reset (:176-190) of one instance, or of every instance with inst = -1.  Every instance has its own 50 ms
 * fragment clock: reset() restarts it, so the instance's next fragment ends fragm frames into the next processed block. */
int b200m_ebu_reset (b200m_ebu* h, int32_t inst, void* stream);
/* integr_start / integr_pause (ebu_r128_proc.h:77-78) / integr_reset (.cc:193-204); inst = -1: all */
/* one instance back to its state after init(): integration off, filters, ring, loudness values and histograms cleared; its
 * 50 ms fragment clock keeps running (see b200m_ebu_reset for one that restarts it) */
int b200m_ebu_clear (b200m_ebu* h, int32_t inst, void* stream);
int b200m_ebu_integr_start (b200m_ebu* h, int32_t inst, void* stream);
int b200m_ebu_integr_pause (b200m_ebu* h, int32_t inst, void* stream);
int b200m_ebu_integr_reset (b200m_ebu* h, int32_t inst, void* stream);
/* Ebu_r128_proc::process(nfram, input[]) (:207-248) for every instance. 0 < nfram <= 8192. */
int b200m_ebu_process_device (b200m_ebu* h, const float* d_in, size_t stride, uint32_t nfram, void* stream);
int b200m_ebu_process_host (b200m_ebu* h, const float* in, size_t stride, uint32_t nfram);
/* Ragged blocks: Ebu_r128_proc::process (len[i], rows of i) for every instance i, over the first len[i] <= nfram frames of its
 * rows; len[i] == 0: process is not called for i at all.  len: host array of n_inst; NULL (or every len[i] == nfram) is exactly
 * b200m_ebu_process_*.  Instance i ends up bit-identical to a private Ebu_r128_proc fed only its own len[i] > 0 blocks, in order:
 * its 50 ms fragment clock advances by len[i], not nfram.  Frames at or after len[i] never reach a result (they may hold anything,
 * NaN included).  A len[i] > nfram is B200M_E_INVAL and enqueues nothing.  Controls, snapshots and the whole-mix reduce keep
 * their meaning.  Loudness of many clips of different lengths: feed each clip's frames and a 0 length once it has ended. */
int b200m_ebu_process_ragged_device (b200m_ebu* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream);
int b200m_ebu_process_ragged_host (b200m_ebu* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len);
/* getters -> host array of n_inst results.  stream = the stream last used for processing
 * (ignored after process_host, which uses the bank's stream). */
int b200m_ebu_results (b200m_ebu* h, b200m_ebu_result* out, void* stream);
/* Loudness log (an extension; the reference keeps only the latest values): one point per completed 50 ms fragment of an instance
 * (every pass through process()'s _frcnt == 0 branch, :217-243), holding exactly what b200m_ebu_results would return right after
 * that fragment, its gating included.  Points are written whether integration runs or not; controls write none and leave the log
 * alone, snapshots neither save nor restore it.  Each instance keeps its last `capacity` points in a ring on the device. */
typedef struct b200m_ebu_point { float loudness_M, loudness_S, integrated, range_min, range_max; } b200m_ebu_point;
/* capacity points per instance; 0 turns the log off and frees it; (re)enabling empties it.  B200M_E_NOMEM (the log off) if the
 * device cannot hold 2 x capacity x n_inst points. */
int b200m_ebu_log_enable (b200m_ebu* h, uint32_t capacity, void* stream);
/* the capacity the log was enabled with: the row length of b200m_ebu_log_drain's `out`; 0 while the log is off or h is NULL */
uint32_t b200m_ebu_log_capacity (const b200m_ebu* h);
/* host out [n_inst][capacity], count [n_inst], lost [n_inst]: instance i's points since the previous drain, oldest first, in
 * out[i][0 .. count[i]) (NaN after them); lost[i] older unread points were overwritten.  Ordered after the work on `stream` like
 * b200m_ebu_results (synchronises it).  B200M_E_INVAL with the log off. */
int b200m_ebu_log_drain (b200m_ebu* h, b200m_ebu_point* out, uint32_t* count, uint64_t* lost, void* stream);
/* histogram_M()/histogram_S() (:91-92) of one instance: 751 + 751 int32 */
int b200m_ebu_histogram (b200m_ebu* h, uint32_t inst, int32_t* hist_M, int32_t* hist_S, void* stream);
/* K-weighting coefficients as designed on the host (detect_init, :263-293): a0 a1 a2 b1 b2 c3 c4 */
size_t b200m_ebu_snapshot_size (b200m_ebu* h);                          /* see b200m_r128_snapshot */
int b200m_ebu_snapshot (b200m_ebu* h, void* buf, size_t bytes, void* stream);
int b200m_ebu_restore (b200m_ebu* h, const void* buf, size_t bytes, void* stream);
int b200m_ebu_coeffs (const b200m_ebu* h, float out7[7]);
/* internal state of one instance for differential tests: z[nchan][4], power ring[64], frpwr,
 * counters {frcnt, wrind, div1, div2}, all the instance's own */
int b200m_ebu_state (b200m_ebu* h, uint32_t inst, float* z, float* power64, float* frpwr, int32_t counters4[4], void* stream);
/* Whole-mix gated loudness (an extension; the reference has no cross-instance quantity):
 * sums hist_M/hist_S/counts of all instances on the device into d_out[2*752+...]; the caller
 * may all-reduce that int32 vector across GPUs (NCCL) and hand it to b200m_ebu_mix_finish. */
#define B200M_MIX_WORDS 1508      /* histM[752] histS[752] cntM cntS errM errS */
int b200m_ebu_mix_reduce (b200m_ebu* h, int32_t* d_out, void* stream);
/* calc_integ + calc_range (:105-150) on a summed histogram vector (device pointer);
 * out5 (host) = integrated, integ_thr, range_min, range_max, range_thr */
int b200m_ebu_mix_finish (b200m_ebu* h, const int32_t* d_mix, float out5[5], void* stream);
/* Album loudness (an extension; the reference has no album concept): the whole-mix quantity for many groups of instances at once,
 * e.g. the albums, playlists or segmented episodes of a library metered clip by clip.  An album's histograms are the sum of its
 * members' histograms, i.e. the union of their 400 ms and 3 s measurement blocks (no block spans two clips, so this is not the
 * loudness of the clips played back to back; it is libebur128's loudness_global_multiple).
 * b200m_ebu_group_reduce: group (host, n_inst entries) maps instance i to album group[i] in 0 .. n_groups - 1, or to
 * B200M_NO_GROUP (counted in no album).  d_out (device) receives n_groups rows of B200M_MIX_WORDS int32, each in the layout of
 * b200m_ebu_mix_reduce's vector; an album without members gets a zero row.  n_groups does not depend on n_inst: shards of one
 * library reduce into the same shape, which may be all-reduced across GPUs (int32 sums) and handed to b200m_ebu_group_finish.
 * The member list is uploaded again only when group differs from the previous call's.
 * b200m_ebu_group_finish: calc_integ + calc_range (:105-150) on each of the n_groups rows of d_groups (device); out5 (host,
 * n_groups x 5) = integrated, integ_thr, range_min, range_max, range_thr of each row, -200 where the reference reports nothing (an
 * empty album among them).  One device-to-host copy and one synchronisation per call.
 * Both are ordered like the getters (an EBU bank of an EBUr128 bank follows that bank's path) and write nothing the bank's
 * processing reads.  B200M_E_INVAL, with nothing enqueued, for a NULL argument, n_groups == 0,
 * n_groups > B200M_MAX_GROUPS, or a group[i] >= n_groups other than B200M_NO_GROUP.  The sums are exact while each album's block
 * counts fit in int32, as for b200m_ebu_mix_reduce. */
#define B200M_NO_GROUP   0xFFFFFFFFu
#define B200M_MAX_GROUPS 65536u     /* 395 MB of d_out */
int b200m_ebu_group_reduce (b200m_ebu* h, const uint32_t* group, uint32_t n_groups, int32_t* d_out, void* stream);
int b200m_ebu_group_finish (b200m_ebu* h, const int32_t* d_groups, uint32_t n_groups, float* out5, void* stream);

/* ======================================================================================
 * True-peak + K-meter bank — replaces LV2M::TruePeakdsp (jmeters/truepeakdsp.h:28-61) and
 * LV2M::Kmeterdsp (jmeters/kmeterdsp.h:27-62), one mono meter of each kind per channel, as
 * driven by dr14_run in TPnRMS mode (src/dr14.c:391-394,425-450), dbtp_run / kmeter_run
 * (src/meters.cc:333-508) and ebur128_run's dBTP option (src/ebulv2.cc:344-347,360-367).
 * ====================================================================================== */
typedef struct b200m_tpk b200m_tpk;

#define B200M_TPK_TRUEPEAK 1u     /* run TruePeakdsp per channel */
#define B200M_TPK_KMETER   2u     /* run Kmeterdsp per channel   */
#define B200M_TP_MODE_PROCESS 0u  /* TruePeakdsp::process      (:41-99)  */
#define B200M_TP_MODE_MAX     1u  /* TruePeakdsp::process_max  (:101-124) */

typedef struct b200m_tpk_result {
    float tp_m, tp_p;             /* TruePeakdsp::read(m,p) (:133-138) — linear */
    float km_rms, km_peak;        /* Kmeterdsp::read(rms,peak) (kmeterdsp.cc:150-155) — linear */
} b200m_tpk_result;

int b200m_tpk_create (b200m_tpk** out, int device, uint32_t n_chan, float fsamp, uint32_t flags);
int b200m_tpk_destroy (b200m_tpk* h);
/* process() of every enabled meter over one block; tp_mode selects process / process_max */
int b200m_tpk_process_device (b200m_tpk* h, const float* d_in, size_t stride, uint32_t nfram, uint32_t tp_mode, void* stream);
int b200m_tpk_process_host (b200m_tpk* h, const float* in, size_t stride, uint32_t nfram, uint32_t tp_mode);
/* Ragged process() blocks: channel i runs TruePeakdsp::process (:41-99) and Kmeterdsp::process (kmeterdsp.cc:65-140) over the first
 * len[i] <= nfram frames of its row only, bit-identical to a private meter fed only those frames.  len: host array of n_chan.
 * - Frames at or after len[i] may hold anything, NaN and Inf included: they reach no state and no reading.
 * - len[i] == 0: the channel is not called: no process, no end-of-block scrub or bias; b200m_tpk_read_device after this block leaves
 *   its reading and read latch alone.
 * - A length above nfram returns B200M_E_INVAL and enqueues nothing.
 * - NULL, or every len[i] == nfram, is exactly b200m_tpk_process_* (tp_mode process(): same kernels, launches and bits).
 * - Controls, path switches and streams are ordered between ragged blocks as between plain ones.
 * A ragged block always runs the exact 16-channel process() kernel, whatever B200M_TPK_SPLIT, B200M_TPK_WIDE, B200M_TPK_DEC or the
 * precision mode select for plain blocks: in a B200M_PREC_FMA bank its readings are exact for that block.  Ragged process_max blocks:
 * b200m_r128_run_ragged_*. */
int b200m_tpk_process_ragged_device (b200m_tpk* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream);
int b200m_tpk_process_ragged_host (b200m_tpk* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len);
/* Arithmetic of the 4x polyphase FIR (zita-resampler/resampler.cc:213-230).
 *   B200M_PREC_EXACT (default): the reference's operation order, unfused -- every float bit-identical to the reference build.
 *   B200M_PREC_FMA: fused multiply-add accumulation using the table's symmetry, phase 0 taken as the pure delay it is to
 *     7.7e-16: 2.4x fewer instructions; true-peak / dBTP readings stay within +-1e-4 dB of the reference,
 *     the K-meter and every integer result are unaffected.  Default can be preset with B200M_TPK_PRECISION=fma. */
enum { B200M_PREC_EXACT = 0, B200M_PREC_FMA = 1 };
int b200m_tpk_set_precision (b200m_tpk* h, int mode);
int b200m_tpk_precision (const b200m_tpk* h);
/* read() of every enabled meter (sets TruePeakdsp::_res / Kmeterdsp::_flag) */
int b200m_tpk_read_device (b200m_tpk* h, void* stream);
int b200m_tpk_results (b200m_tpk* h, b200m_tpk_result* out, void* stream);
/* TruePeakdsp::reset (:140-145) / Kmeterdsp::reset (kmeterdsp.cc:157-162); chan = -1: all */
int b200m_tpk_reset (b200m_tpk* h, int32_t chan, void* stream);
/* reset() plus zero ballistics filters and oversampler history: the channel as a newly constructed meter leaves init(); chan = -1: all */
int b200m_tpk_clear (b200m_tpk* h, int32_t chan, void* stream);
/* Kmeterdsp::reset of every channel only (reset_peaks of the TPnRMS / DR14 plugin, src/dr14.c:241-258) */
int b200m_tpk_reset_kmeter (b200m_tpk* h, void* stream);
/* host-designed constants: w[4] = w1 w2 w3 g (truepeakdsp.cc:153-157); ctab[120] = zita table
 * (zita-resampler/resampler-table.cc:52-75, hl=24 np=4 fr=1); km[2] = omega, (float)hold */
size_t b200m_tpk_snapshot_size (b200m_tpk* h);                          /* see b200m_r128_snapshot */
int b200m_tpk_snapshot (b200m_tpk* h, void* buf, size_t bytes, void* stream);
int b200m_tpk_restore (b200m_tpk* h, const void* buf, size_t bytes, void* stream);
int b200m_tpk_coeffs (const b200m_tpk* h, float w[4], float ctab[120], float km[2]);
/* internal state for differential tests, arrays of n_chan: tp {m,p,z1,z2,res}, km [n][8] as
 * z1 z2 rms peak fall cnt fpp flag */
int b200m_tpk_state (b200m_tpk* h, float* tp_m, float* tp_p, float* tp_z1, float* tp_z2, int32_t* tp_res, float* km8, void* stream);
/* the raw 4x oversampled stream of the LAST processed block of one channel (4*nfram floats),
 * only kept when enabled with b200m_tpk_debug_capture(h,1): FIR bit-exactness tests */
int b200m_tpk_debug_capture (b200m_tpk* h, int enable);
int b200m_tpk_debug_upsampled (b200m_tpk* h, uint32_t chan, float* out, uint32_t n_out, void* stream);
/* launch timeline of the opt-in slab pipeline (B200M_TPK_SPLIT=2 with B200M_TPK_TIMELINE=1): up to n slots of
 * {first CTA start, last CTA end} in %globaltimer ns, two slots (filter, ballistics) per slab; returns the count, -1 = off */
int b200m_tpk_debug_timeline (b200m_tpk* h, unsigned long long* out, int n);

/* ======================================================================================
 * EBUr128 plugin cycle — the audio part of ebur128_run (src/ebulv2.cc:341-367) for N stereo
 * instances: Ebu_r128_proc::process + (if dbtp_enable) TruePeakdsp::process_max on both channels,
 * the getters, and the dBTP hold  tp_max = max (tp_max, coef_to_db (max (tp0, tp1)))  (:227-230,360-367).
 * b200m_r128_create_nch: the same cycle for instances of 1..5 channels (the maximum of the reads of all
 * the instance's channels, taken before coef_to_db).
 * One host->device copy per block feeds both meters.  Atom/radar/GUI messaging is out of scope.
 * ====================================================================================== */
typedef struct b200m_r128 b200m_r128;
enum { B200M_R128_START = 1, B200M_R128_PAUSE = 2, B200M_R128_RESET = 3, B200M_R128_CLEAR_TPMAX = 4, B200M_R128_CLEAR = 5, B200M_R128_NEW = 6 };
/* START/PAUSE/RESET: CTL_START/PAUSE/RESET, src/uris.h:187-203; RESET = ebu_reset (src/ebulv2.cc:45-61): integr_reset + tp_max hold cleared.
 * CLEAR_TPMAX: the hold alone (a dBTP-disabled cycle, :365-366).
 * CLEAR (inst >= 0): one slot back to a freshly created instance -- EBU state, true-peak histories and hold -- its 50 ms fragment
 *   clock running on.
 * NEW (inst >= 0): CLEAR with the instance's own fragment clock restarted: a freshly instantiated plugin whose first run() is the
 *   next block (b200m_ebu_reset of the instance). */
int b200m_r128_create (b200m_r128** out, int device, uint32_t n_inst, float fsamp, int dbtp_enable);
/* n_inst instances of nchan = 1..5 channels (b200m_r128_create: nchan = 2).  Input rows are inst * nchan + c, channels in
 * Ebu_r128_proc's order L R C Ls Rs (gains 1 1 1 1.41 1.41, ebumeter/ebu_r128_proc.cc:29); LFE is not an input (BS.1770 leaves
 * it out): pass the non-LFE rows.  Every other b200m_r128_* call works on such a bank; CLEAR / NEW and a disabled dBTP cover all
 * the instance's channels, and a snapshot restores only into a bank with the same nchan. */
int b200m_r128_create_nch (b200m_r128** out, int device, uint32_t n_inst, uint32_t nchan, float fsamp, int dbtp_enable);
/* Immersive and custom layouts: n_inst instances of nchan = 1..32 channels with per-channel loudness weights gains[c]
 * (b200m_ebu_create_weighted; b200m_bs1770_weights gives the BS.1770-4 weights of a layout).  Rows are inst * nchan + c.  A gain
 * of 0 keeps a channel out of the loudness but not out of the dBTP hold: pass an LFE row in place to get BS.1770 loudness and the
 * true peak of every channel.  The reference's weights for 1..5 channels give exactly b200m_r128_create_nch's bank (same kernels
 * and snapshot bytes).  Every other b200m_r128_* call works on such a bank unchanged; its snapshot restores only into a bank with
 * the same nchan and gains. */
int b200m_r128_create_weighted (b200m_r128** out, int device, uint32_t n_inst, uint32_t nchan, const float* gains, float fsamp, int dbtp_enable);
int b200m_r128_destroy (b200m_r128* h);
int b200m_r128_control (b200m_r128* h, int32_t inst, int cmd, void* stream);      /* inst = -1: all */
int b200m_r128_run_device (b200m_r128* h, const float* d_in, size_t stride, uint32_t nfram, void* stream);
int b200m_r128_run_host (b200m_r128* h, const float* in, size_t stride, uint32_t nfram);
/* Ragged blocks: the EBUr128 cycle of instance i over its first len[i] <= nfram frames -- Ebu process (len[i]), process_max
 * (len[i]) on each of its channels, the reads and the tp_max hold; len[i] == 0: the plugin did not run this cycle (no process,
 * no read, hold unchanged).  len: host array of n_inst; NULL (or every len[i] == nfram) is exactly b200m_r128_run_* (same kernels,
 * launches and bits).  Parity, unread frames and B200M_E_INVAL as for b200m_ebu_process_ragged_*; a dBTP-disabled instance stays
 * frozen whatever its length.  A ragged block runs the chunk-parallel true-peak FIR in either precision mode, never the
 * tensor-core or fused kernels. */
int b200m_r128_run_ragged_device (b200m_r128* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream);
int b200m_r128_run_ragged_host (b200m_r128* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len);
/* ebu_out: n_inst getter blocks (may be NULL); tp_max_db: n_inst floats, -inf when dBTP is disabled (may be NULL) */
int b200m_r128_results (b200m_r128* h, b200m_ebu_result* ebu_out, float* tp_max_db, void* stream);
/* self->dbtp_enable (CTL_UISETTINGS bit 64, src/ebulv2.cc:316-317): the true-peak meters only run while enabled; while
 * disabled tp_max is -inf every cycle (:365-366).  Takes effect with the next run. */
int b200m_r128_set_dbtp (b200m_r128* h, int enable);
/* the same switch for one instance (inst = -1: every instance, = b200m_r128_set_dbtp).  A disabled instance's two TruePeakdsp
 * histories stay frozen, its tp_max is -inf after every cycle, and its first block after re-enabling reads the samples that
 * preceded the disable.  A bank whose instances all share one setting launches nothing extra; a mixed one adds one small kernel
 * per cycle. */
int b200m_r128_set_dbtp_inst (b200m_r128* h, int32_t inst, int enable);
/* precision of the true-peak FIR (b200m_tpk_set_precision); Ebu_r128_proc's arithmetic is always exact */
int b200m_r128_set_precision (b200m_r128* h, int mode);
/* histogram_M() / histogram_S() of one instance (src/ebulv2.cc:425-429), ordered after the bank's last run */
int b200m_r128_histogram (b200m_r128* h, uint32_t inst, int32_t* hist_M, int32_t* hist_S, void* stream);
/* Checkpoint / resume (new: the reference saves only UI settings, never DSP state -- src/ebulv2.cc:513-548): the complete
 * state of the bank (filters, 64-fragment rings, both histograms of every instance, gating clocks, true-peak histories and
 * holds) as one host blob.  restore() needs a bank created with the same n_inst / fsamp; processing then continues
 * bit-identically to the bank the snapshot was taken from.  Also available per bank: b200m_ebu_* / b200m_tpk_*. */
size_t b200m_r128_snapshot_size (b200m_r128* h);
int b200m_r128_snapshot (b200m_r128* h, void* buf, size_t bytes, void* stream);
int b200m_r128_restore (b200m_r128* h, const void* buf, size_t bytes, void* stream);
/* True-peak curves (an extension, like the loudness log): the loudness log of b200m_r128_ebu (h) with a sixth field per point, the
 * dBTP of its fragment: coef_to_db (:227-230) of the largest |4x oversampled| output that TruePeakdsp::process_max computes, over
 * all the instance's channels (zero-weight ones included, as in the tp_max hold) and the input frames of that fragment that ran
 * with the instance's dBTP on (b200m_r128_set_dbtp_inst; in a ragged block its first len[i] frames).  -inf when that maximum is 0 or
 * no frame of the fragment ran with dBTP on.  The fragment is the one the loudness fields describe: the frames between two edges of
 * the instance's 50 ms clock, across blocks.
 * - The frames of the fragment left open by a control that restarts or clears the instance's clock (NEW, CLEAR, b200m_ebu_reset /
 *   b200m_ebu_clear of the member) or by a restore do not count: the first point after it covers only the frames metered since.
 *   RESET and CLEAR_TPMAX leave the fragment alone.
 * - While the plane is on, the cycle's true-peak maximum runs on the chunk-parallel kernel in either precision mode, never on the
 *   tensor-core or fused kernels (its tolerance-mode readings are those of a B200M_TPK_TC=0 bank); B200M_TPK_CHUNKED=0 does not apply.
 *   With the plane off nothing changes. */
typedef struct b200m_r128_point { float loudness_M, loudness_S, integrated, range_min, range_max, dbtp; } b200m_r128_point;
/* the loudness log with the dBTP plane, as b200m_ebu_log_enable (b200m_r128_ebu (h), capacity, stream) otherwise: 0 turns both off,
 * (re)enabling empties the log (the first point's dBTP then covers the frames metered from here on), B200M_E_NOMEM leaves it off.
 * B200M_E_UNSUPPORTED below 5120 Hz (fragments of < 256 frames).
 * b200m_ebu_log_enable on the member bank turns the plane off. */
int b200m_r128_log_enable (b200m_r128* h, uint32_t capacity, void* stream);
/* b200m_ebu_log_drain of the member bank with the sixth field: out [n_inst][capacity] (b200m_ebu_log_capacity), the same read
 * cursor, ordering and NaN past count.  B200M_E_INVAL while the plane is off (b200m_ebu_log_drain still drains five fields then). */
int b200m_r128_log_drain (b200m_r128* h, b200m_r128_point* out, uint32_t* count, uint64_t* lost, void* stream);
b200m_ebu* b200m_r128_ebu (b200m_r128* h);     /* the underlying banks (histograms, state, coefficients) */
/* the EBU bank of an EBUr128 bank follows that bank's path: after a b200m_r128_run_host* call its getters, controls and log calls
 * (b200m_ebu_log_enable / _drain) run on the EBUr128 bank's own stream, after a device-path call on the stream they are given */
b200m_tpk* b200m_r128_tpk (b200m_r128* h);

/* ======================================================================================
 * DR-14 / TPnRMS bank (SURVEY §8f rank 2) — replaces dr14_run (src/dr14.c:354-482) for n_inst instances of
 * n_channels (1 or 2): Kmeterdsp::process + TruePeakdsp::process + read() per channel and, with dr_mode, the 3 s
 * window statistics of dr14_calc_rms_score (:285-352).  The result block mirrors the plugin's output ports
 * (DRPortIndex :27-43): all values in dB as the reference writes them.  Every instance has its own 3 s window phase,
 * which restarts when that instance is reset, so each instance behaves as a plugin of its own.  dr_mode needs
 * rate >= 2731 Hz (a window longer than the largest block).
 * ====================================================================================== */
typedef struct b200m_dr14 b200m_dr14;
typedef struct b200m_dr14_result {
    float v_rms[2], v_peak[2];       /* *p_v_rms = coeff_to_db (km rms), *p_v_peak = coeff_to_db (true-peak ballistic m) (:430-431) */
    float m_peak[2], m_rms[2];       /* coeff_to_db (max true peak) (:432); DR mode: top-20 % RMS score, else coeff_to_db (km peak) (:444-446) */
    float dr[2], dr_total;           /* DR mode: per channel and averaged, clamped to 1..20; 21 = not yet valid (:436-458) */
    float block_count;               /* 3.0 * num_fragments (:460) */
} b200m_dr14_result;
int b200m_dr14_create (b200m_dr14** out, int device, uint32_t n_inst, uint32_t n_channels, double rate, int dr_mode);
int b200m_dr14_destroy (b200m_dr14* h);
int b200m_dr14_run_device (b200m_dr14* h, const float* d_in, size_t stride, uint32_t nfram, void* stream);   /* rows: inst * n_channels + c */
int b200m_dr14_run_host (b200m_dr14* h, const float* in, size_t stride, uint32_t nfram);
/* Ragged blocks: instance i runs dr14_run over the first len[i] <= nfram frames of its rows, bit-identical to a private plugin
 * instance fed only those frames (DR-14 and TPnRMS mode, mono and stereo, device and host path).  len: host array of n_inst.
 * - Frames at or after len[i] may hold anything, NaN and Inf included: they reach no result and no state.  A window that the
 *   instance's frames do not complete is not scored, as the reference never scores a track's partial last window.
 * - len[i] == 0: the instance is not called at all: no process and no read() (the meters' read latches stay), its result row and
 *   m_dbtp are unchanged, and its 3 s window clock does not advance.
 * - A length above nfram returns B200M_E_INVAL and enqueues nothing.
 * - NULL, or every len[i] == nfram, is exactly b200m_dr14_run_* (same kernels, launches and bits).
 * - Controls, path switches and streams are ordered between ragged blocks as between plain ones.
 * A ragged block always runs the exact fused process() kernel (whatever B200M_TPK_SPLIT / B200M_TPK_WIDE select for plain blocks),
 * plus one clock kernel in DR mode. */
int b200m_dr14_run_ragged_device (b200m_dr14* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream);
int b200m_dr14_run_ragged_host (b200m_dr14* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len);
int b200m_dr14_reset (b200m_dr14* h, void* stream);                                       /* reset_peaks, every instance */
/* B200M_DR14_RESET: reset_peaks (:246-262) of the listed instances: K-meter reset, m_peak = m_rms = -81, m_dbtp = 0, window
 * sums, second-peak pair, histogram, num_fragments, and the instance's 3 s window restarts with the next block.
 * B200M_DR14_CLEAR: the instance as a freshly instantiated plugin (:139-165): RESET plus b200m_tpk_clear of its channels.
 * inst = NULL, count = 0: every instance; a listed instance may repeat.  One upload and two kernels per call, ordered with the
 * bank's runs on the stream the bank currently runs on. */
enum { B200M_DR14_RESET = 1, B200M_DR14_CLEAR = 2 };
int b200m_dr14_control (b200m_dr14* h, const uint32_t* inst, uint32_t count, int cmd, void* stream);
int b200m_dr14_results (b200m_dr14* h, b200m_dr14_result* out, void* stream);
int b200m_dr14_histogram (b200m_dr14* h, uint32_t inst, uint32_t chan, uint32_t* hist8000, void* stream);   /* hist[c] (:46,309-311) */
/* Window log (an extension; the reference keeps only the latest values), DR mode: one point per completed 3 s window of an
 * instance (every dr14_calc_rms_score call, :285-352), silent windows included.  All fields float, in dB unless noted:
 * - window: the windows this instance completed since its last RESET / CLEAR / creation, this one included (1, 2, ...); window k
 *   ends after frame k * (n_sample_cnt + 1) of the instance's own frames.  Exact up to 2^24 windows.
 * - silent: 1 if the silence gate skipped the window (:287-298): no histogram entry, the running fields unchanged; else 0.
 * - rms: the window's RMS as the reference bins it, coeff_to_db (sqrt (2 rms_sum / n_sample_cnt)) (:306,310).  -80 for a silent
 *   window, which is also what that formula gives for it (a window whose sum is NaN is silent too).
 * - peak: coeff_to_db (peak_cur) handed to the second-peak pair (:338-344): the largest sample (signed maximum, as the reference)
 *   since the previous scored window or reset.  NaN for a silent window, whose samples count towards the next scored one's peak.
 * - m_rms, dr, dr_total, block_count: the b200m_dr14_results fields after this window, bit for bit (a window is longer than any
 *   block, so at most one closes per block).  peak2: coeff_to_db of the second-highest window peak after this window, -81 before
 *   3 scored windows (not the m_peak port, which is the true-peak hold).
 * - A mono bank's channel-1 fields and dr_total are NaN.
 * A ragged block logs a window only if it closes within the instance's len[i] frames, as it is scored.  RESET / CLEAR drop the open
 * window (no point for it; window restarts at 1) and leave the points already logged; no control writes a point. */
typedef struct b200m_dr14_point {
    float window, silent;
    float rms[2], peak[2];
    float m_rms[2], peak2[2];
    float dr[2], dr_total, block_count;
} b200m_dr14_point;
/* capacity points per instance, kept in a ring on the device; 0 turns the log off and frees it; (re)enabling empties it.
 * B200M_E_NOMEM (the log off) if the device cannot hold 2 x capacity x n_inst points; B200M_E_UNSUPPORTED in TPnRMS mode. */
int b200m_dr14_log_enable (b200m_dr14* h, uint32_t capacity, void* stream);
/* the capacity the log was enabled with: the row length of b200m_dr14_log_drain's `out`; 0 while the log is off or h is NULL */
uint32_t b200m_dr14_log_capacity (const b200m_dr14* h);
/* host out [n_inst][capacity], count [n_inst], lost [n_inst]: instance i's points since the previous drain, oldest first, in
 * out[i][0 .. count[i]) (NaN after them); lost[i] older unread points were overwritten.  Ordered after the work on `stream` like
 * b200m_dr14_results (synchronises it).  B200M_E_INVAL with the log off. */
int b200m_dr14_log_drain (b200m_dr14* h, b200m_dr14_point* out, uint32_t* count, uint64_t* lost, void* stream);
/* Album DR (an extension; the reference has no album concept), DR mode: the DR score of many groups of instances at once, e.g. the
 * albums of a library metered track by track, bit-identical to one private dr14 instance fed every member track back to back when
 * each track holds whole 3 s windows and ends in a scored one.  dr14_calc_rms_score (:285-352) depends only on the 8000-bin RMS
 * histogram, the count of scored windows and the two highest window peaks, so an album's state is the sum of its members'
 * histograms and window counts and the two largest of their top-two peak pairs.
 * b200m_dr14_group_reduce: group (host, n_inst entries) maps instance i to album group[i] in 0 .. n_groups - 1, or to
 * B200M_NO_GROUP, as for b200m_ebu_group_reduce.  d_rows (device) receives n_groups rows of B200M_DR14_GROUP_WORDS (nch) int32:
 * the channel-0 histogram, then the channel-1 histogram (bins in the order of b200m_dr14_histogram), the number of windows scored
 * (the sum of the members' num_fragments) and the number of members.  The rows are zeroed and summed into with integer atomics,
 * so the rows of shards of one library may be all-reduced with SUM across GPUs.  d_peaks (device) receives [n_groups][nch][3]
 * floats of linear values: the album's highest and second-highest window peak (the top two of the members' peak_hist pairs by
 * value; NaN never enters a pair) and its true-peak hold (m_dbtp, the m_peak port before coeff_to_db): the largest member hold
 * that is not NaN, NaN only if every member's hold is NaN (MAX written as `>` makes a hold NaN after a block whose true peak is, :430).  Peaks cannot be
 * summed: shards all-gather theirs and hand every part to the finish.  An album without members gets zeros everywhere, which is
 * what a freshly instantiated plugin holds.
 * b200m_dr14_group_finish: d_peaks (device) holds n_parts consecutive [n_groups][nch][3] blocks (one per shard after an
 * all-gather; n_parts = 1 on one GPU).  Per album the finish merges the parts' top-two pairs by value and takes their largest
 * non-NaN hold (an empty part holds 0), then scores each channel's row as dr14_calc_rms_score does: m_cut = MAX (1, floorf (nf /
 * 5.0)), the walk from the top bin down in the reference's bin order, nothing before nf > 2 windows, coeff_to_db; then the port
 * arithmetic (:436-460).  out (host, n_groups entries): m_rms, dr, dr_total, block_count as in b200m_dr14_result; peak2 as in
 * b200m_dr14_point; m_peak = coeff_to_db (hold); windows and members as floats (exact up to 2^24).  A mono bank's channel-1
 * fields and dr_total are NaN.  An empty album reads like a fresh plugin: m_rms = peak2 = -81, dr = dr_total = 21,
 * block_count 0, m_peak -80.  One device-to-host copy and one synchronisation per call.
 * Both are ordered like the getters and write nothing the bank's processing reads.  B200M_E_INVAL, with nothing enqueued, for a
 * NULL argument, n_groups == 0, n_groups > B200M_DR14_MAX_GROUPS, n_parts == 0, or a group[i] >= n_groups other than
 * B200M_NO_GROUP; B200M_E_UNSUPPORTED on a TPnRMS bank.  The sums are exact while each album's window counts fit in int32. */
#define B200M_DR14_MAX_GROUPS 16384u                          /* 1.05 GB of d_rows for a stereo bank */
#define B200M_DR14_GROUP_WORDS(nch) ((nch) * 8000u + 2u)      /* int32 words per album row */
typedef struct b200m_dr14_album {
    float m_rms[2], peak2[2];        /* top-20 % RMS score and second-highest window peak (dB, -81 before 3 windows) */
    float dr[2], dr_total;           /* clamped to 1..20; 21 = not valid */
    float block_count;               /* 3.0 * windows */
    float m_peak[2];                 /* coeff_to_db of the largest member true-peak hold */
    float windows, members;
} b200m_dr14_album;
int b200m_dr14_group_reduce (b200m_dr14* h, const uint32_t* group, uint32_t n_groups, int32_t* d_rows, float* d_peaks, void* stream);
int b200m_dr14_group_finish (b200m_dr14* h, const int32_t* d_rows, const float* d_peaks, uint32_t n_parts, uint32_t n_groups,
                             b200m_dr14_album* out, void* stream);

/* ======================================================================================
 * Stereo correlation bank — replaces LV2M::Stcorrdsp (jmeters/stcorrdsp.h:27-55) as driven by
 * cor_run (src/meters.cc:511-536) and xfer_run (src/xfer.c:248-251).
 * ====================================================================================== */
typedef struct b200m_cor b200m_cor;
int b200m_cor_create (b200m_cor** out, int device, uint32_t n_inst, int fsamp, float flp, float tcf);
int b200m_cor_destroy (b200m_cor* h);
int b200m_cor_process_device (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, void* stream);
int b200m_cor_process_host (b200m_cor* h, const float* in, size_t stride, uint32_t nfram);
int b200m_cor_results (b200m_cor* h, float* out, void* stream);           /* Stcorrdsp::read (:79-82) */
/* pair inst (-1: all) back to a newly constructed Stcorrdsp (stcorrdsp.cc:33-37): the five filter states and the reading zero, in
 * both precision modes, and, while the histogram plane is on (b200m_cor_hist_enable), its counts and sum.  Ordered with the bank's
 * runs on the stream it currently runs on.  A phasewheel ring fed from this bank (b200m_pw_attach_cor) is not touched. */
int b200m_cor_clear (b200m_cor* h, int32_t inst, void* stream);
/* b200m_cor_process_* with a per-pair hold: run = n_inst flags, NULL = every pair runs (exactly b200m_cor_process_*).  A pair
 * with run[i] == 0 is left as if the call had not been made for it: its five filter states and its reading stay bit-identical,
 * without the end-of-process scrub and bias, and its input rows are not read (they may hold anything, NaN included).  Each pair's
 * arithmetic is independent of its neighbours', so the others advance exactly as in a bank called only in their own active
 * cycles, in both precision modes.  The mask is uploaded only when it differs from the previous call's. */
int b200m_cor_process_ctl_device (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, const uint8_t* run, void* stream);
int b200m_cor_process_ctl_host (b200m_cor* h, const float* in, size_t stride, uint32_t nfram, const uint8_t* run);
/* Ragged blocks: pair i runs Stcorrdsp::process (:47-77) over the first len[i] <= nfram frames of its rows only, as a private
 * Stcorrdsp fed only those frames (bit-identical in B200M_PREC_EXACT, within 1e-5 in B200M_PREC_FMA, bit-identical there too when
 * tcf * fsamp > 21600: see b200m_cor_set_precision).  len: host array of n_inst.
 * - Frames at or after len[i] may hold anything, NaN and Inf included: they reach no state and no reading.
 * - len[i] == 0: the pair is not called (exactly the hold of b200m_cor_process_ctl_*, which is this call with run[i] ? nfram : 0).
 * - A length above nfram returns B200M_E_INVAL and enqueues nothing.
 * - NULL, or every len[i] == nfram, is exactly b200m_cor_process_* (same kernels, launches and bits).
 * - The lengths are uploaded only when they differ from the previous call's.
 * - A bank attached to a phasewheel bank (b200m_pw_attach_cor) returns B200M_E_UNSUPPORTED: the phasewheel ring advances bank-wide.
 *   b200m_pw_attach_cor (pw, NULL) detaches it. */
int b200m_cor_process_ragged_device (b200m_cor* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream);
int b200m_cor_process_ragged_host (b200m_cor* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len);
/* B200M_PREC_EXACT (default): the five recurrences run serially in time, one lane per pair, bit-identical to the reference.
 * B200M_PREC_FMA: time-parallel evaluation -- the recurrences are linear one-pole filters, so a warp owns ONE pair, its lanes take
 * consecutive time segments and an affine warp scan stitches them: 32x more parallelism for small banks (2048 pairs are 64 warps
 * in exact mode); the correlation stays within 1e-5 of the reference.  The reference's own fp32 rounding noise grows with the product
 * filters' memory tcf * fsamp, and no more accurate evaluation can follow it: a bank whose memory exceeds 21600 samples (tcf 0.3 s
 * above 72 kHz, i.e. at 88.2-192 kHz; tcf above 0.45 s at 48 kHz) runs the exact kernel in this mode too, bit-identical to the
 * reference.  The bound is fixed at creation, whatever the block.  While the correlation histogram plane is on
 * (b200m_cor_hist_enable) this mode also runs the exact kernel: the plane has one form, and the plane, the states and the readings
 * are then bit-identical to B200M_PREC_EXACT. */
int b200m_cor_set_precision (b200m_cor* h, int mode);
int b200m_cor_state (b200m_cor* h, float* state5, void* stream);          /* [n][5] zl zr zlr zll zrr */
int b200m_cor_coeffs (const b200m_cor* h, float w[2]);
/* Correlation histogram (an extension; the reference keeps only the state its read() reports at block end): with the plane on,
 * after each frame's five updates of Stcorrdsp::process (stcorrdsp.cc:58-62) every pair forms the frame's reading
 * r = zlr / sqrtf (zll * zrr + 1e-10f) (the read() formula, :79-82, on the in-loop state; fp32, no contraction).  The frame counts
 * if zll + zrr >= thr (fp32) and r is finite, with thr = (float) (2 * 10^(gate_db / 10)) computed in double.  A counted frame adds
 * 1 to bin clamp ((int) floorf ((r + 1.0f) * 100.0f), 0, 199) of the pair's B200M_COR_HIST_BINS bins of width 0.01 over [-1, 1]
 * (r = 1 falls in bin 199; readings past +-1 are clamped), and adds (double) r to the pair's double sum in frame order.  The
 * end-of-process scrub and bias (:65-75) apply at block end only, as without the plane.  Ragged blocks and held pairs of
 * b200m_cor_process_ctl_* add only the frames the pair runs; a phasewheel bank's feed (b200m_pw_attach_cor) counts like a call of
 * this bank.  Ports and b200m_cor_state are bit-identical with the plane on or off; with it off the bank runs exactly the kernels it
 * runs without it.
 * enable != 0: allocates the plane on first use (B200M_E_NOMEM if the device cannot hold 1608 bytes per pair), zeroes every pair's
 * counts and sum, also when it was on already, and sets the gate; 0: stops counting and keeps the memory.  gate_db = -INFINITY
 * gives thr = 0 (every frame with a finite reading counts); NaN or +INFINITY returns B200M_E_INVAL.  While the plane is on,
 * b200m_cor_clear also zeroes the cleared pairs' counts and sums.  Ordered like the getters. */
#define B200M_COR_HIST_BINS 200
int b200m_cor_hist_enable (b200m_cor* h, int enable, float gate_db, void* stream);
/* host counts [n_inst][B200M_COR_HIST_BINS] and sums [n_inst] of every pair, in one copy and one synchronisation of the stream,
 * ordered like b200m_cor_results; the mean reading of the counted frames is sums / (the row's total count).  B200M_E_INVAL while
 * the plane is off. */
int b200m_cor_hist_read (b200m_cor* h, uint64_t* counts, double* sums, void* stream);

/* ======================================================================================
 * Needle-meter ballistics bank (SURVEY §8f rank 3) — replaces LV2M::Vumeterdsp (jmeters/vumeterdsp.cc:45-93),
 * Iec1ppmdsp / Iec2ppmdsp (jmeters/iec1ppmdsp.cc, iec2ppmdsp.cc :47-99) and Msppmdsp (jmeters/msppmdsp.cc:50-143)
 * as driven by run() and bbcm_run() (src/meters.cc:298-331,552-589).
 * kind VU / IEC1 / IEC2: n_units mono meters (row i = meter i).  kind MS: n_units stereo pairs (rows 2i, 2i+1),
 * two meters per pair, M = processM at index 2i, S = processS at index 2i+1.
 * ====================================================================================== */
typedef struct b200m_ppm b200m_ppm;
enum { B200M_PPM_VU = 0, B200M_PPM_IEC1 = 1, B200M_PPM_IEC2 = 2, B200M_PPM_MS = 3 };
int b200m_ppm_create (b200m_ppm** out, int device, uint32_t n_units, float fsamp, int kind);
int b200m_ppm_destroy (b200m_ppm* h);
int b200m_ppm_set_gain (b200m_ppm* h, float db_m, float db_s);       /* Msppmdsp::set_gain of the M and S meters (default -6, -6) */
/* Msppmdsp::set_gain (msppmdsp.cc:135-143) of one pair's M and S meters (unit = -1: every pair, exactly b200m_ppm_set_gain).  The
 * gains are designed on the host, skipped per meter when the dB value is unchanged, and reach the bank with its next process call,
 * on that call's stream. */
int b200m_ppm_set_gain_inst (b200m_ppm* h, int32_t unit, float db_m, float db_s);
/* unit (-1: all) back to newly constructed meters (vumeterdsp.cc / iec1ppmdsp.cc / iec2ppmdsp.cc / msppmdsp.cc constructors):
 * z1 z2 m = 0, _res = true, both meters of an M/S pair, whose gains return to -6 / -6 dB, and, while the histogram plane is on
 * (b200m_ppm_hist_enable), the unit's counts and statistics (both rows of an M/S pair).  Ordered with the bank's runs on the
 * stream it currently runs on. */
int b200m_ppm_clear (b200m_ppm* h, int32_t unit, void* stream);
int b200m_ppm_process_device (b200m_ppm* h, const float* d_in, size_t stride, uint32_t nfram, void* stream);
int b200m_ppm_process_host (b200m_ppm* h, const float* in, size_t stride, uint32_t nfram);
/* Ragged blocks: unit u (a meter, or for B200M_PPM_MS a stereo pair and its two meters) runs process() (vumeterdsp.cc:45-77,
 * iec1ppmdsp.cc / iec2ppmdsp.cc :47-80, msppmdsp.cc:50-118) over the first len[u] <= nfram frames of its rows only, bit-identical to a
 * private meter fed only those frames.  len: host array of n_units.
 * - Frames at or after len[u] may hold anything, NaN and Inf included: they reach no state and no reading.
 * - len[u] == 0: the unit is not called: no clamp, scrub or bias, _res unchanged; b200m_ppm_read_device after this block leaves its
 *   reading and _res alone.  M/S gains set in between (b200m_ppm_set_gain_inst) apply from the unit's next call, as on a private meter.
 * - A length above nfram returns B200M_E_INVAL and enqueues nothing.
 * - NULL, or every len[u] == nfram, is exactly b200m_ppm_process_* (same kernels, launches and bits).
 * - Controls, path switches and streams are ordered between ragged blocks as between plain ones. */
int b200m_ppm_process_ragged_device (b200m_ppm* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream);
int b200m_ppm_process_ragged_host (b200m_ppm* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len);
int b200m_ppm_read_device (b200m_ppm* h, void* stream);                /* read(): _res = true, value = _g * _m */
int b200m_ppm_results (b200m_ppm* h, float* out, void* stream);        /* one float per meter */
int b200m_ppm_state (b200m_ppm* h, float* state4, void* stream);       /* per meter: z1 z2 m res */
int b200m_design_ppm (int kind, float fsamp, float w[4]);              /* w1 w2 w3 g (VU: w 0 0 g) */
/* Needle histogram (an extension; read() keeps only the highest needle since the last read): process() meters a call in groups of
 * 4 frames ("n /= 4": a call's last nfram mod 4 frames are not metered).  With the plane on, after each group's updates every meter
 * takes the needle value s the reference compares with m (VU: z2 after its update, vumeterdsp.cc:57-68; IEC I / IEC II and both
 * meters of an M/S pair: t = z1 + z2, iec1ppmdsp.cc / iec2ppmdsp.cc / msppmdsp.cc) and forms the group's reading v = _g * s (fp32,
 * no contraction): the value read() would return if that group alone had set _m.  Per meter the plane keeps:
 * - counts [B200M_PPM_HIST_BINS] (uint64): a finite v goes to bin #{k : v >= e[k]}, with the 241 edges
 *   e[k] = (float) pow (10.0, (-80.0 + 0.5 * k) / 20.0) (double, k = 0..240, b200m_ppm_hist_edges).  Bin 0 holds readings below
 *   -80 dB (v <= 0 included: a VU needle can swing negative), bins 1..240 are 0.5 dB wide, bin 241 is +40 dB and above;
 * - nonfinite: groups whose v is not finite (IEC on Inf input, VU on NaN or Inf input); they go to no bin;
 * - peak: the largest finite v, -INFINITY before the first;
 * - overs of the bank's limit L = (float) pow (10.0, limit_db / 20.0) (double): over_groups counts finite v >= L, overs the runs of
 *   such readings, longest_over the most over readings in one run (the open run included) and run the open run's length (0 if the
 *   last finite reading was not over).  A non-finite reading neither starts, extends nor ends a run; a run continues across calls,
 *   ragged zero-length holds and unmetered tails, as on a private meter fed the clip in pieces.
 * Ragged blocks count only each unit's own groups; a unit with length 0 adds nothing.  Ports and b200m_ppm_state are bit-identical
 * with the plane on or off; with it off the bank runs exactly the kernels it runs without it. */
#define B200M_PPM_HIST_BINS 242
typedef struct {
    uint64_t nonfinite, over_groups, overs, longest_over, run;
    float peak;
    uint32_t pad;
} b200m_ppm_hist_stats;
/* enable != 0: allocates the plane on first use (B200M_E_NOMEM if the device cannot hold 1984 bytes per meter), zeroes every
 * meter's counts and statistics (peak -INFINITY), also when it was on already, and sets L; 0: stops counting and keeps the memory.
 * limit_db NaN returns B200M_E_INVAL; +INFINITY (no reading is over) and -INFINITY (L = 0) are allowed.  Ordered like the getters. */
int b200m_ppm_hist_enable (b200m_ppm* h, int enable, float limit_db, void* stream);
/* host counts [n_meters][B200M_PPM_HIST_BINS] and stats [n_meters], in one copy and one synchronisation of the stream, ordered like
 * b200m_ppm_results.  B200M_E_INVAL while the plane is off. */
int b200m_ppm_hist_read (b200m_ppm* h, uint64_t* counts, b200m_ppm_hist_stats* stats, void* stream);
/* the library's 241 bin edges e[k] (host only: needs no device), so that callers bin with the same floats */
int b200m_ppm_hist_edges (float* edges);

/* True-peak / K-meter histogram (an extension of the b200m_tpk bank above; read() keeps only the highest value since the last read).
 * With the plane on, every channel keeps a TP row (with B200M_TPK_TRUEPEAK) and a KM row (with B200M_TPK_KMETER): counts
 * [B200M_PPM_HIST_BINS] (uint64) and a b200m_ppm_hist_stats, with the needle plane's edges e[k] (b200m_ppm_hist_edges) and rules: a
 * finite reading u goes to bin #{k : u >= e[k]}; nonfinite counts the others; peak is the largest finite u (-INFINITY before the
 * first); over_groups counts readings u >= L, overs their runs, longest_over the longest run (the open run included) and run the open
 * run.  A non-finite reading neither starts, extends nor ends a run; runs continue across calls, ragged zero-length holds and the
 * K-meter's unmetered nfram mod 4 tails.
 * - TP: one reading per frame of TruePeakdsp::process (truepeakdsp.cc:57-84): u = the largest of the frame's four |out|, the values
 *   the reference compares in "if (v > p) p = v"; a frame with a non-finite |out| is nonfinite.  With a read() after every block,
 *   the finite frames' maximum in a block is that block's tp_p; a clip with no non-finite frame has peak = the _p of a meter never
 *   read over it.
 * - KM: one reading per group of 4 frames of Kmeterdsp::process (kmeterdsp.cc:80-98): after the group's z2 update, u = sqrtf (2 * z2)
 *   (fp32, correctly rounded, no contraction), the rms the block end would form (:109) had the block ended there; a NaN z2 (which the
 *   block end scrubs to 0) or a non-finite u is nonfinite.  L_km is dBFS RMS on the port's sine-calibrated scale.
 * - L_tp = (float) pow (10.0, tp_limit_db / 20.0), L_km likewise from km_limit_db (double), per bank.
 * Only process() blocks count, plain and ragged: a ragged row counts its own first len[i] frames, length 0 adds nothing.  While the
 * plane is on every process() block runs the exact 16-channel kernel, whatever B200M_TPK_SPLIT, B200M_TPK_WIDE, B200M_TPK_DEC or
 * the precision mode select: in a B200M_PREC_FMA bank the plane, the states and the readings are exact for those blocks.  Ports and
 * b200m_tpk_state are bit-identical with the plane on or off; with it off the bank runs exactly the kernels it runs without it.
 * process_max with the plane on returns B200M_E_UNSUPPORTED and enqueues nothing.  b200m_tpk_clear also zeroes the cleared
 * channels' rows; b200m_tpk_reset, b200m_tpk_reset_kmeter and b200m_tpk_read_device leave the plane alone.  The plane is not part of
 * b200m_tpk_snapshot, and b200m_tpk_restore leaves its rows as they are. */
/* enable != 0: allocates the plane on first use (B200M_E_NOMEM if the device cannot hold it: 1984 bytes per channel and meter),
 * zeroes every row (peak -INFINITY), also when it was on already, and sets both limits; 0: stops counting and keeps the memory.  A
 * NaN limit returns B200M_E_INVAL; +-INFINITY is allowed.  The true-peak bank of an EBUr128 bank (b200m_r128_tpk) returns
 * B200M_E_UNSUPPORTED.  Ordered like the getters. */
int b200m_tpk_hist_enable (b200m_tpk* h, int enable, float tp_limit_db, float km_limit_db, void* stream);
/* host counts [n_chan][B200M_PPM_HIST_BINS] and stats [n_chan] of each meter the bank has, in one copy and one synchronisation of
 * the stream; the pointers of a meter the bank lacks must be NULL.  B200M_E_INVAL while the plane is off. */
int b200m_tpk_hist_read (b200m_tpk* h, uint64_t* tp_counts, b200m_ppm_hist_stats* tp_stats, uint64_t* km_counts,
                         b200m_ppm_hist_stats* km_stats, void* stream);

/* ======================================================================================
 * Bit-meter and signal-distribution-histogram banks (SURVEY §8f rank 1), N mono instances each.
 * bit-meter: float_stats + the acquisition / ~5 fps window logic of bim_run (src/bitmeter.c:63-105,248-327);
 *   results = int32 histS[584] (layout src/uris.h:52-60), counters {zero,pos,nan,inf,den}, {min,max}, integration time.
 * SigDistHist: the sample loop of sdh_run (src/sigdistlv2.c:287-327): int32 histS[361], {max count, peak bin},
 *   {sum, running mean, running variance accumulator} in double, integration time.
 * Controls mirror the plugins' CTL_* messages (src/uris.h:187-203).  Every instance has its own control state on the device:
 *   bit-meter: integrating, averaging, integration time (capped at 2^31 samples) and the ~5 fps window clock, so its window
 *   closes, publishes and (windowed mode) clears independently of the others; SigDistHist: integrating, integration time.
 * b200m_*_control_inst acts on one instance (inst >= 0) or on all (inst = -1: exactly b200m_*_control).  Controls are ordered
 * with the bank's runs on the stream the bank currently runs on.
 * B200M_CTL_CLEAR turns an instance into a freshly instantiated plugin: bit-meter = bim_reset, integrating, windowed, window
 * clock 0, empty published snapshot (src/bitmeter.c:146-158); SigDistHist = sdh_reset with integration off (src/sigdistlv2.c:141-150).
 * ====================================================================================== */
typedef struct b200m_bim b200m_bim;
typedef struct b200m_sdh b200m_sdh;
enum { B200M_CTL_START = 1, B200M_CTL_PAUSE = 2, B200M_CTL_RESET = 3, B200M_CTL_AVERAGE = 4, B200M_CTL_WINDOWED = 5, B200M_CTL_CLEAR = 6 };
int b200m_bim_create (b200m_bim** out, int device, uint32_t n_inst, double rate);
int b200m_bim_destroy (b200m_bim* h);
int b200m_bim_control (b200m_bim* h, int cmd, void* stream);                      /* every instance */
int b200m_bim_control_inst (b200m_bim* h, int32_t inst, int cmd, void* stream);   /* inst = -1: every instance */
int b200m_bim_run_device (b200m_bim* h, const float* d_in, size_t stride, uint32_t nfram, void* stream);
int b200m_bim_run_host (b200m_bim* h, const float* in, size_t stride, uint32_t nfram);
int b200m_bim_results (b200m_bim* h, uint32_t inst, int32_t* hist584, int32_t* cnt5, float* minmax2, int64_t* integration_time, void* stream);
/* 1 if the last run closed a ~5 fps window (self->radar_resync >= fps_limit, src/bitmeter.c:264-267,293); the statistics
 * as they stood at that moment -- what bim_run publishes in its bim_stats message before the windowed-mode bim_clear
 * (:269-291,323-325) -- stay readable through b200m_bim_published until the next window closes.
 * b200m_bim_window_closed follows a bank-wide window clock: it is exact for a bank whose instances were only cleared together
 * (b200m_bim_control, or b200m_bim_control_inst with inst = -1) and driven only with plain blocks.  A ragged block (below) does not
 * advance that clock, and b200m_bim_window_closed reads 0 after one.  The closed flag of each instance's own clock is returned by
 * b200m_bim_results_all. */
int b200m_bim_window_closed (const b200m_bim* h);
int b200m_bim_published (b200m_bim* h, uint32_t inst, int32_t* hist584, int32_t* cnt5, float* minmax2, int64_t* integration_time, void* stream);
/* every instance in ONE synchronisation, ordered after the bank's last run; any pointer may be NULL.  Row layouts, n = n_inst:
 *   hist [n][584]       the live histogram (src/uris.h:52-60)
 *   cnt5 [n][5]         zero, pos, nan, inf, den
 *   minmax2 [n][2]      min, max of |sample| over normal numbers
 *   integration_time [n]
 *   closed [n]          1 if the last run closed that instance's window (0 after a ragged block with len[i] == 0)
 *   pub_* [n][...]      the same rows for the snapshot published when that instance's window last closed */
int b200m_bim_results_all (b200m_bim* h, int32_t* hist, int32_t* cnt5, float* minmax2, int64_t* integration_time, int32_t* closed,
                           int32_t* pub_hist, int32_t* pub_cnt5, float* pub_minmax2, int64_t* pub_integration_time, void* stream);
int b200m_sdh_create (b200m_sdh** out, int device, uint32_t n_inst, double rate);
int b200m_sdh_destroy (b200m_sdh* h);
int b200m_sdh_control (b200m_sdh* h, int cmd, void* stream);                      /* every instance; START PAUSE RESET CLEAR */
int b200m_sdh_control_inst (b200m_sdh* h, int32_t inst, int cmd, void* stream);   /* inst = -1: every instance */
int b200m_sdh_run_device (b200m_sdh* h, const float* d_in, size_t stride, uint32_t nfram, void* stream);
int b200m_sdh_run_host (b200m_sdh* h, const float* in, size_t stride, uint32_t nfram);
int b200m_sdh_results (b200m_sdh* h, uint32_t inst, int32_t* hist361, int32_t* max_peak2, double* avg_tmp_var3, int64_t* integration_time, void* stream);
/* every instance in ONE synchronisation; any pointer may be NULL.  Rows: hist [n][361], max_peak2 [n][2] = max count, peak bin;
 * avg_tmp_var3 [n][3] = sum, running mean, running variance accumulator; integration_time [n] */
int b200m_sdh_results_all (b200m_sdh* h, int32_t* hist, int32_t* max_peak2, double* avg_tmp_var3, int64_t* integration_time, void* stream);
/* Ragged blocks: instance i runs bim_run (src/bitmeter.c:248-327) / sdh_run (src/sigdistlv2.c:287-327) over the first len[i] <= nfram
 * frames of its row only, bit-identical to a private plugin instance fed only those frames: histograms, counters, min / max, the fp64
 * accumulators and the integration time (its 2^31-sample cap tested against len[i]).  len: host array of n_inst.
 * - Frames at or after len[i] may hold anything, NaN, Inf and denormals included: they reach no counter, bin or statistic.
 * - The bit-meter's ~5 fps window limit is that of a run of len[i] frames, len[i] * ceil (rate / (5 * len[i])) (:264), and its window
 *   clock advances by len[i].
 * - len[i] == 0: the instance is not run: nothing is acquired, its window clock stands still, no result changes -- except the
 *   bit-meter's closed flag of that instance in b200m_bim_results_all, which reads 0 (its window did not close in this block).
 * - A ragged bit-meter block leaves the bank-wide clock of b200m_bim_window_closed alone; that function reads 0 after it.
 * - A length above nfram returns B200M_E_INVAL and enqueues nothing.
 * - NULL, or every len[i] == nfram, is exactly b200m_bim_run_* / b200m_sdh_run_* (same kernels, launches and bits).
 * - Controls, path switches and streams are ordered between ragged blocks as between plain ones. */
int b200m_bim_run_ragged_device (b200m_bim* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream);
int b200m_bim_run_ragged_host (b200m_bim* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len);
int b200m_sdh_run_ragged_device (b200m_sdh* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream);
int b200m_sdh_run_ragged_host (b200m_sdh* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len);

/* ======================================================================================
 * 30-band 1/3-octave spectrum bank — replaces spectrum_instantiate / spectrum_run
 * (src/spectrumlv2.c:73-121,159-257) over bandpass_setup / bandpass_process (src/spectr.c:68-206).
 * ====================================================================================== */
typedef struct b200m_spec b200m_spec;
int b200m_spec_create (b200m_spec** out, int device, uint32_t n_inst, uint32_t nchan, double rate);
int b200m_spec_destroy (b200m_spec* h);
/* one spectrum_run(): speed = *port 60, reset = *port 61 (same value for every instance) */
int b200m_spec_process_device (b200m_spec* h, const float* d_in, size_t stride, uint32_t nfram, float speed, float reset, void* stream);
int b200m_spec_process_host (b200m_spec* h, const float* in, size_t stride, uint32_t nfram, float speed, float reset);
/* one spectrum_run() with every instance's own controls: ctl = host array [n_inst][2] = {*port 60, *port 61} of this cycle.  Each
 * instance keeps its own speed / reset handshake state (src/spectrumlv2.c:170-205), fall-off coefficient and `ac` dither phase;
 * the two calls above are this one with the same pair for every instance.  Only instances whose run parameters changed are
 * uploaded, on the call's stream. */
int b200m_spec_process_ctl_device (b200m_spec* h, const float* d_in, size_t stride, uint32_t nfram, const float* ctl, void* stream);
int b200m_spec_process_ctl_host (b200m_spec* h, const float* in, size_t stride, uint32_t nfram, const float* ctl);
/* Ragged blocks: instance i runs spectrum_run (src/spectrumlv2.c:159-257) over the first len[i] <= nfram frames of its rows only, with
 * its controls ctl[i], as a private plugin instance fed only those frames (ports bit-identical in B200M_PREC_EXACT, within +-1e-4 dB
 * in B200M_PREC_FMA).  len: host array of n_inst; ctl as for b200m_spec_process_ctl_*.
 * - Frames at or after len[i] may hold anything, NaN and Inf included: they reach no state and no port.
 * - len[i] == 0: the instance is not run: its ports, filters and speed / reset handshake state stay, its ctl row is ignored.
 * - Each instance's `ac` dither phase follows its own frame count.
 * - A length above nfram returns B200M_E_INVAL and enqueues nothing.
 * - NULL, or every len[i] == nfram, is exactly b200m_spec_process_ctl_* (same kernels, launches and bits).
 * - Controls, path switches and streams are ordered between ragged blocks as between plain ones. */
int b200m_spec_process_ragged_device (b200m_spec* h, const float* d_in, size_t stride, uint32_t nfram, const float* ctl, const uint32_t* len,
                                      void* stream);
int b200m_spec_process_ragged_host (b200m_spec* h, const float* in, size_t stride, uint32_t nfram, const float* ctl, const uint32_t* len);
/* instance inst (-1: all) back to what b200m_spec_create gives (spectrum_instantiate, src/spectrumlv2.c:73-121): filter states,
 * val, max and ports zero, rst_h = -4, spd_h = 1, `ac` restarting with the next frame.  Ordered with the bank's runs on the stream
 * it currently runs on. */
int b200m_spec_clear (b200m_spec* h, int32_t inst, void* stream);
/* B200M_PREC_EXACT (default): the reference's fp64 rounding sequence, ports bit-identical.  B200M_PREC_FMA: fused multiply-adds in the
 * biquad cascade (25 instead of 39 fp64 instructions per frame and band); band levels within +-1e-4 dB. */
int b200m_spec_set_precision (b200m_spec* h, int mode);
/* ports 0..59 of every instance: 30 band levels (dB), 30 band maxima (dB) */
int b200m_spec_results (b200m_spec* h, float* out60, void* stream);
int b200m_spec_state (b200m_spec* h, uint32_t inst, double* z360, float* val30, float* max30, void* stream);
int b200m_spec_coeffs (const b200m_spec* h, double* W1080);              /* [30][6][6] a0 a1 a2 b0 b1 b2 */
/* Long-term average spectrum (an extension; the reference keeps only the smoothed level and its peak hold): with the plane on, every
 * band of every instance adds its per-frame power s = v * v (the value spectrum_run smooths, src/spectrumlv2.c:221-226, after
 * bandpass_process, src/spectr.c:79-87) to a double sum, sum = sum + (double) s frame by frame in frame order, and counts the frames
 * it added.  A frame whose s is not finite adds nothing and is not counted (non-finite input leaves the filters NaN until the
 * end-of-run scrub, :229-236).  Ragged blocks add an instance's own len[i] frames only; B200M_PREC_FMA adds its own v.  Ports and
 * b200m_spec_state are bit-identical with the plane on or off; with it off the bank runs exactly the kernel it runs without it.
 * enable != 0: allocates the plane on first use (B200M_E_NOMEM if the device cannot hold 16 x 32 bytes per instance) and zeroes every
 * instance's sums and counts, also when it was on already; 0: turns it off.  While it is on, b200m_spec_clear also zeroes the
 * cleared instances' sums and counts.  Ordered like the getters. */
int b200m_spec_ltas_enable (b200m_spec* h, int enable, void* stream);
/* host sums [n_inst][30] and counts [n_inst][30] of every instance, in one copy and one synchronisation of the stream, ordered like
 * b200m_spec_results; the band's long-term average power is sums / counts.  B200M_E_INVAL while the plane is off. */
int b200m_spec_ltas_read (b200m_spec* h, double* sums, uint64_t* counts, void* stream);

/* ======================================================================================
 * Phasewheel FFT analysis bank — replaces fftx_init / fftx_run / ft_analyze (gui/fft.c:208-361)
 * for both channels plus process_audio (gui/phasewheel.c:1307-1342).
 * ====================================================================================== */
typedef struct b200m_pw b200m_pw;
/* fft_bins: the GUI's selector values (gui/phasewheel.c:1108-1116): 64, 128, ... 8192 and 6144 (window = 2 * fft_bins) */
int b200m_pw_create (b200m_pw** out, int device, uint32_t n_inst, uint32_t fft_bins, double rate);
int b200m_pw_destroy (b200m_pw* h);
/* which GUI's process_audio follows the FFTs: PHASEWHEEL (default; phase difference, level, peak: gui/phasewheel.c:1307-1342)
 * or STEREOSCOPE (gui/stereoscope.c:705-741: smoothed lr[] returned in `phase`, smoothed level[]; db_thresh fixed at 1e-20,
 * no peak; the reference GUI defaults to fft_bins 512).  Re-initialises the outputs like the GUI's reinitialize_fft. */
enum { B200M_PW_PHASEWHEEL = 0, B200M_PW_STEREOSCOPE = 1 };
int b200m_pw_set_mode (b200m_pw* h, int mode);
/* returns (via *fired) whether this call completed an analysis (fftx_run()==0) */
int b200m_pw_process_device (b200m_pw* h, const float* d_in, size_t stride, uint32_t nfram, float db_thresh, int* fired, void* stream);
int b200m_pw_process_host (b200m_pw* h, const float* in, size_t stride, uint32_t nfram, float db_thresh, int* fired);
/* Ragged blocks: stereo instance i (rows 2i, 2i+1) runs fftx_run on both channels (gui/fft.c:296-361) and then process_audio over the
 * first len[i] <= nfram frames of its rows only, with its own ring offset and 25 Hz analysis clock, bit-identical to a private bank of
 * one fed only those frames: phase, level, peak and the b200m_pw_raw spectra.  len: host array of n_inst.  *fired is 1 if any instance
 * completed an analysis in this call.
 * - Frames at or after len[i] may hold anything, NaN and Inf included: they reach no ring, spectrum or output.
 * - len[i] == 0: the instance is not called: its ring and clock do not advance and its outputs stay.
 * - A length above nfram returns B200M_E_INVAL and enqueues nothing.
 * - NULL, or every len[i] == nfram, is exactly b200m_pw_process_* (same kernels, launches and bits) while the instances share one
 *   ring offset and clock.  Once ragged blocks have moved them apart, plain blocks run the per-instance form with every length nfram
 *   (unfused from an attached correlation bank), until the offsets and clocks agree again.
 * - An attached correlation bank (b200m_pw_attach_cor) runs each pair over the same len[i] frames (b200m_cor_process_ragged_*), once
 *   per call; b200m_cor_process_ragged_* on that bank itself stays refused.
 * - Controls, path switches and streams are ordered between ragged blocks as between plain ones. */
int b200m_pw_process_ragged_device (b200m_pw* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len,
                                    float db_thresh, int* fired, void* stream);
int b200m_pw_process_ragged_host (b200m_pw* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len,
                                  float db_thresh, int* fired);
/* phase[n_inst][fft_bins], level[n_inst][fft_bins], peak[n_inst] (ui->phase/level/peak) */
int b200m_pw_results (b200m_pw* h, float* phase, float* level, float* peak, void* stream);
/* ft->power / ft->phase of both channels of the last analysis (gui/fft.c:163-180), kept only while b200m_pw_debug_capture is on */
int b200m_pw_debug_capture (b200m_pw* h, int enable);
int b200m_pw_raw (b200m_pw* h, uint32_t inst, float* powL, float* powR, float* phL, float* phR, void* stream);
/* Fused feed: with a correlation bank of n_inst pairs attached, b200m_pw_process_* also runs Stcorrdsp::process of that bank on the
 * same block (what xfer_run does per cycle, src/xfer.c:248-251) in ONE kernel that reads the input once: the block is staged in
 * shared memory for the correlation recurrences and appended to the FFT ring from there.  Read the correlation with
 * b200m_cor_results; do not call b200m_cor_process_* on an attached bank.  cor = NULL detaches. */
int b200m_pw_attach_cor (b200m_pw* h, b200m_cor* cor);
/* Cross-spectrum plane (an extension; the reference keeps only the last analysis's spectra): with the plane on, every analysis of an
 * instance adds, for every bin k = 0 .. fft_bins-1, four terms to its row sums[inst][term][k] (fp64):
 *   B200M_PW_XSPEC_LL  |L_k|^2,   B200M_PW_XSPEC_RR  |R_k|^2,   B200M_PW_XSPEC_RL_RE  Re (R_k conj L_k),   B200M_PW_XSPEC_RL_IM  Im (R_k conj L_k)
 * L_k, R_k: the fp32 spectra the analysis forms (gui/fft.c:163-180; bin fft_bins-1 as every other bin, though its ports read 0).
 * Each term is formed in double from the fp32 parts (exact products, one rounding) and added in analysis order, so atan2 (RL_IM, RL_RE)
 * has the phasewheel's sign, arg R - arg L (gui/phasewheel.c:1323-1325).  counts[inst][0] counts the analyses added.  An analysis with a
 * non-finite Re / Im part in either spectrum adds nothing and counts in counts[inst][1] (skipped) instead; it does not depend on db_thresh.
 * - Every analysis counts, not only the last of a call, whose spectra alone reach the ports: a firing of the 25 Hz clock before the
 *   last one of a call runs a plane-only analysis.  With blocks of at most ceil (rate / 25) frames a call fires at most once and the
 *   plane adds no launch.
 * - Ports, peak, b200m_pw_raw and the stereoscope smoothing are bit-identical with the plane on or off, in both modes; with it off
 *   the bank runs exactly the kernels it runs without it.
 * - Ragged blocks add an instance's own analyses only; the fused correlation feed and ragged blocks accumulate exactly as unfused
 *   and plain blocks do.  b200m_pw_set_mode, b200m_pw_debug_capture and b200m_pw_attach_cor leave the plane alone.
 * enable != 0: allocates the plane on first use (B200M_E_NOMEM if the device cannot hold 32 fft_bins + 16 bytes per instance) and zeroes
 * every row and count, also when it was on already; 0: stops accumulating and keeps the memory.  Ordered like the getters. */
#define B200M_PW_XSPEC_TERMS 4
enum { B200M_PW_XSPEC_LL = 0, B200M_PW_XSPEC_RR = 1, B200M_PW_XSPEC_RL_RE = 2, B200M_PW_XSPEC_RL_IM = 3 };
int b200m_pw_xspec_enable (b200m_pw* h, int enable, void* stream);
/* host sums [n_inst][4][fft_bins] and counts [n_inst][2] (analyses, skipped), in one copy and one synchronisation of the stream,
 * ordered like b200m_pw_results.  B200M_E_INVAL while the plane has never been enabled. */
int b200m_pw_xspec_read (b200m_pw* h, double* sums, uint64_t* counts, void* stream);
/* device pointers of the result planes, for callers that keep the spectra on the GPU */
int b200m_pw_device_results (b200m_pw* h, const float** d_phase, const float** d_level, const float** d_peak);

/* ======================================================================================
 * PCM input: interleaved integer or float PCM, as a file decodes (frames [t][c], little-endian), to the planar float32 rows every
 * bank reads, on the device.  Clip i of n_clips starts at in + i * in_stride (bytes) and holds nfram frames of nchan samples; out row
 * k = i * nchan + c (at out + k * out_stride floats), frame t, is the sample at in + i * in_stride + (t * nchan + c) * bps, scaled by
 * 2^-(bits - 1), the normalised float read of integer PCM (-full scale reads -1.0):
 *   B200M_PCM_S16  2 bytes   (float) x * 2^-15, exact
 *   B200M_PCM_S24  3 bytes   packed, sign-extended 24-bit x, (float) x * 2^-23, exact
 *   B200M_PCM_S32  4 bytes   x rounded to the nearest float (ties to even), times 2^-31 (exact): INT32_MAX reads 1.0f
 *   B200M_PCM_F32  4 bytes   a bit copy: NaN payloads, +-Inf, -0 and denormals kept
 * One launch, asynchronous on `stream`; in and out must not overlap.  in and in_stride must be multiples of the sample size (any
 * byte for S24, so a WAV data chunk can be converted where it lies).  B200M_E_INVAL, with nothing enqueued: a NULL pointer, an
 * unknown format, n_clips == 0, nchan outside 1..B200M_PCM_MAX_CHANNELS, nfram outside 1..B200M_MAX_BLOCK, in_stride < nfram *
 * nchan * bps, a misaligned in or in_stride, out_stride < nfram.  No CUDA device: B200M_E_NODEVICE.  A host caller uploads the raw
 * bytes itself (pinned memory: b200m_host_alloc) and converts them here.
 * ====================================================================================== */
enum { B200M_PCM_S16 = 0, B200M_PCM_S24 = 1, B200M_PCM_S32 = 2, B200M_PCM_F32 = 3 };
#define B200M_PCM_MAX_CHANNELS 32u   /* the widest instance any bank meters: the weighted EBUr128 bank */
int b200m_pcm_planar_device (int device, const void* in, int format, uint32_t n_clips, uint32_t nchan, uint32_t nfram,
                             size_t in_stride, float* out, size_t out_stride, void* stream);

/* ======================================================================================
 * LV2 facade: the library also exports `lv2_descriptor (index)` (the one symbol of the reference's meters.so,
 * src/meters.cc:739-792) serving all 38 plugin URIs.  b200m_lv2_gon_layout lists, for tests, the offsets of the goniometer
 * instance struct that the reference GUI reads through instance-access (src/goniometer.h:113-169): rb, ui_active,
 * rb_overrun, s_sfact, s_linewidth, input, rate, ntfy, msg_thread_lock, map, sizeof; returns how many there are.
 * ====================================================================================== */
int b200m_lv2_gon_layout (size_t* out, int n);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* B200METERS_H */
