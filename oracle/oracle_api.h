/* oracle_api.h — C API shared by the two CPU oracles of this repo.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product:
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * `--impl reference` leg may load these libraries, and only as the checker
 * (or as the timed CPU baseline), never as the thing shipped.
 *
 * Two shared objects export exactly this API:
 *   oracle/_ref/libmeters_ref.so   kind "reference": the UNMODIFIED reference
 *        sources compiled by path from /root/reference (oracle/Makefile),
 *        driven through thin extern "C" shims (oracle/ref_wrap.cc).
 *   oracle/liboracle_port.so       kind "port": a from-scratch CPU restatement
 *        of the same algorithms (oracle/oracle_port.cc), each function citing
 *        the reference file:line it follows.  It is pinned against the
 *        reference build and the committed golden vectors by tests/.
 *
 * Layout convention for every process call: channel k (k = inst*nchan + c)
 * starts at  in + k*stride  and holds nfram float32 samples (planar audio,
 * as an LV2 host hands it to run(), src/meters.cc:257-296).
 */
#ifndef B200M_ORACLE_API_H
#define B200M_ORACLE_API_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

const char* orc_kind (void);            /* "reference" | "port" */
int         orc_hw_threads (void);

/* ---- EBU R128  (ebumeter/ebu_r128_proc.h:66-125) ---- */
void* orc_ebu_create  (int n_inst, int nchan, float fsamp);
void  orc_ebu_destroy (void* h);
void  orc_ebu_integr  (void* h, int inst, int cmd);   /* 0 pause 1 start 2 reset; inst<0 = all */
void  orc_ebu_reset   (void* h, int inst);             /* Ebu_r128_proc::reset */
void  orc_ebu_process (void* h, const float* in, size_t stride, int nfram, int nthreads);
void  orc_ebu_read    (void* h, float* out);           /* [n_inst][9] M maxM S maxS I Ithr Rmin Rmax Rthr */
void  orc_ebu_hist    (void* h, int inst, int* histM, int* histS, int* counts4); /* 751,751,{cntM,cntS,errM,errS} */
void  orc_ebu_coeffs  (void* h, float* out7);          /* a0 a1 a2 b1 b2 c3 c4 */
void  orc_ebu_state   (void* h, int inst, float* z, float* power64, float* frpwr, int* counters4);
                       /* z: [nchan][4]; counters: frcnt wrind div1 div2 */
/* Ebu_r128_hist::calc_integ + calc_range (:105-150) on caller-given counts: 751 bins and the count word of each
 * histogram.  out5 = integrated, integ_thr, range_min, range_max, range_thr, all pre-set to -200 (what a reset
 * instance reports: calc_integ leaves the threshold unchanged below 50 points).  The range walks have no upper
 * bound: the caller guarantees that the bins sum to the count word and that both walks end by bin 750. */
void  orc_ebu_hist_calc (const int* histM751, int cntM, const int* histS751, int cntS, float* out5);

/* ---- True peak (jmeters/truepeakdsp.h:28-61), one mono meter per channel ---- */
void* orc_tp_create   (int n, float fsamp);
void  orc_tp_destroy  (void* h);
void  orc_tp_process  (void* h, const float* in, size_t stride, int nfram, int mode, int nthreads);
                       /* mode 0: process()   mode 1: process_max() */
void  orc_tp_read     (void* h, float* m, float* p);   /* TruePeakdsp::read(m,p) for every meter */
void  orc_tp_peek     (void* h, float* m, float* p, float* z1, float* z2, int* res); /* no side effect */
void  orc_tp_reset    (void* h, int inst);
void  orc_tp_coeffs   (void* h, float* w4, float* ctab120); /* w1 w2 w3 g ; resampler table (np+1)*hl */
/* raw 4x stream of a fresh meter (after init's pre-roll): out has 4*n floats */
void  orc_tp_upsample (float fsamp, const float* in, int n, int block, float* out);

/* one ebur128_run audio cycle (src/ebulv2.cc:341-347) per stereo instance i: ebu[i].process (L,R) and, if
 * tp != NULL, process_max on tp[2i] (L) and tp[2i+1] (R), followed by read(); all inside ONE thread fan-out
 * and repeated for `nblocks` consecutive blocks (block b starts at in + b*nfram): the CPU baseline of bench.py */
void  orc_r128_cycle  (void* ebu, void* tp, const float* in, size_t stride, int nfram, int nblocks, int nthreads);

/* the EBUr128 PLUGIN itself (kind "reference" only; port returns NULL): n instances driven through ebur128_run,
 * integration started and dBTP enabled as the UI would; out = [n][10]: the nine getters + tp_max (dBTP hold) */
void* orc_ebuplug_create (int n, float rate, int dbtp);
void  orc_ebuplug_destroy (void* h);
void  orc_ebuplug_run (void* h, const float* in, size_t stride, int nfram, int nthreads);
void  orc_ebuplug_read (void* h, float* out10);

/* ---- K-meter (jmeters/kmeterdsp.h:27-62) ---- */
void* orc_km_create   (int n, float fsamp);
void  orc_km_destroy  (void* h);
void  orc_km_process  (void* h, const float* in, size_t stride, int nfram, int nthreads);
void  orc_km_read     (void* h, float* rms, float* peak);        /* Kmeterdsp::read(rms,peak) */
void  orc_km_peek     (void* h, float* state8);                  /* [n][8] z1 z2 rms peak fall cnt fpp flag */
void  orc_km_reset    (void* h, int inst);
void  orc_km_coeffs   (void* h, float* omega, int* hold);

/* ---- needle-meter ballistics (jmeters/vumeterdsp.cc, iec1ppmdsp.cc, iec2ppmdsp.cc, msppmdsp.cc) ----
 * kind 0 VU, 1 IEC type I PPM (DIN/Nordic), 2 IEC type II PPM (BBC/EBU): n mono meters, channel i = row i.
 * kind 3 M/S PPM (BBC M6): n stereo pairs (rows 2i, 2i+1), two meters per pair: M = processM, S = processS */
void* orc_ppm_create  (int n, float fsamp, int kind);
void  orc_ppm_destroy (void* h);
void  orc_ppm_process (void* h, const float* in, size_t stride, int nfram, int nthreads);
void  orc_ppm_read    (void* h, float* out);              /* read(): kind 0-2 [n]; kind 3 [n][2] = M, S */
void  orc_ppm_peek    (void* h, float* state4);           /* per meter z1 z2 m res; kind 3: [n][2][4] */
void  orc_ppm_set_gain(void* h, float db_m, float db_s);  /* kind 3: Msppmdsp::set_gain of the M and S meters */
void  orc_ppm_coeffs  (void* h, float* w4);               /* w1 w2 w3 g   (VU: w, 0, 0, g) */

/* ---- Stereo correlation (jmeters/stcorrdsp.h:27-55) ---- */
void* orc_cor_create  (int n, int fsamp, float flp, float tcf);
void  orc_cor_destroy (void* h);
void  orc_cor_process (void* h, const float* in, size_t stride, int nfram, int nthreads); /* L,R = ch 2i,2i+1 */
void  orc_cor_read    (void* h, float* out);
void  orc_cor_peek    (void* h, float* state5);                  /* [n][5] zl zr zlr zll zrr */
void  orc_cor_coeffs  (void* h, float* w2);

/* ---- 30 band 1/3 octave spectrum (src/spectrumlv2.c:73-257, src/spectr.c:68-206) ---- */
void* orc_spec_create (int n_inst, int nchan, double rate);
void  orc_spec_destroy(void* h);
void  orc_spec_process(void* h, const float* in, size_t stride, int nfram, float speed, float reset, int nthreads);
void  orc_spec_read   (void* h, float* out60);                   /* [n_inst][60]: 30 band dB, 30 max dB (ports 0-59) */
void  orc_spec_state  (void* h, int inst, double* z360, float* val30, float* max30);
void  orc_spec_coeffs (void* h, double* W);                      /* [30][6][6] a0 a1 a2 b0 b1 b2 */

/* ---- bit-meter (src/bitmeter.c: float_stats :63-105, bim_run :181-348), n mono instances ----
 * kind "reference" drives the plugin's own LV2 run(); result fields are read from the instance after each run().
 * average != 0 = CTL_AVERAGE (cumulative); 0 = windowed: statistics are cleared about 5 times per second (:264,325-327) */
void* orc_bim_create  (int n, float rate);
void  orc_bim_destroy (void* h);
void  orc_bim_mode    (void* h, int average, int integrating);
void  orc_bim_process (void* h, const float* in, size_t stride, int nfram, int nthreads);
void  orc_bim_read    (void* h, int inst, int32_t* hist584, int32_t* cnt5, float* minmax2, int64_t* itime); /* cnt5 = zero pos nan inf den */

/* ---- signal distribution histogram (src/sigdistlv2.c: sdh_run :200-396, loop :303-318), n mono instances ---- */
void* orc_sdh_create  (int n, float rate);
void  orc_sdh_destroy (void* h);
void  orc_sdh_integrate (void* h, int on);
void  orc_sdh_process (void* h, const float* in, size_t stride, int nfram, int nthreads);
void  orc_sdh_read    (void* h, int inst, int32_t* hist361, int32_t* maxpeak2, double* avg_tmp_var3, int64_t* itime);

/* DR-14 / TPnRMS: dr14_run (src/dr14.c:354-482) for n instances of nch channels; rows inst*nch + c.
 * read: 12 floats per instance = the output ports v_rms[2] v_peak[2] m_peak[2] m_rms[2] dr[2] dr_total block_count.
 * kind "reference" drives the reference's own dr14 / TPnRMS plugins through LV2 run() (follow-transport off, no atoms). */
void* orc_dr14_create  (int n, int nch, double rate, int dr_mode);
void  orc_dr14_destroy (void* h);
void  orc_dr14_process (void* h, const float* in, size_t stride, int nfram, int nthreads);
void  orc_dr14_reset   (void* h);
void  orc_dr14_read    (void* h, float* out12);

/* ---- phasewheel / stereoscope FFT analysis (gui/fft.c:208-340, gui/phasewheel.c:1307-1342) ----
 * kind "reference" returns NULL from orc_pw_create: FFTW3 is not vendored and absent here. */
void* orc_pw_create   (int n_inst, int fft_bins, double rate);
void  orc_pw_destroy  (void* h);
void  orc_pw_set_mode (void* h, int mode);   /* 0: phasewheel process_audio, 1: stereoscope process_audio (gui/stereoscope.c:705-741; phase[] = lr[]) */
int   orc_pw_process  (void* h, const float* in, size_t stride, int nfram, float db_thresh, int nthreads);
                       /* returns 1 if an analysis fired (all instances are in lock step) */
void  orc_pw_read     (void* h, float* phase, float* level, float* peak); /* [n_inst][fft_bins] x2, [n_inst] */
void  orc_pw_raw      (void* h, int inst, float* powL, float* powR, float* phL, float* phR);

/* ---- the timed CPU baseline (oracle/cpu_bench.inc) ----
 * orc_cpu_info: hardware threads, CPUs in the affinity mask, cgroup CPU quota (0 = none); returns the number of CPUs
 * worth starting a thread on.  orc_r128_bench: `steps` steps of `nblocks` blocks of the EBUr128 audio cycle over n_inst
 * stereo instances on `nthreads` persistent (optionally pinned) workers that own their instances and input;
 * out6 = samples/s, wall s, threads, steps, slowest/mean worker time, samples/s per thread */
int   orc_cpu_info    (int* hw_threads, int* affinity_cpus, double* cgroup_quota_cpus);
long long orc_log10f_check (uint32_t first_bits, uint32_t count, const float* dev, int nthreads, uint32_t* bad3); /* host libm log10f vs dev[i] */
int   orc_r128_bench  (int n_inst, int nfram, int nblocks, int nthreads, int pin, int steps, int warmup, float fsamp, double* out6);

#ifdef __cplusplus
}
#endif
#endif
