// ref_wrap.cc — extern "C" shims (oracle_api.h) over the UNMODIFIED reference classes.
//
// TEST INFRASTRUCTURE ONLY (see oracle_api.h).  This file contains no DSP: every
// sample is processed by the reference's own objects, compiled by path from
// /root/reference by oracle/Makefile into oracle/_ref/ (never copied into the repo):
//   jmeters/{truepeakdsp,kmeterdsp,stcorrdsp}.cc, ebumeter/ebu_r128_proc.cc,
//   zita-resampler/{resampler,resampler-table}.cc, src/spectr.c + src/spectrumlv2.c
// `#define private public` around the reference headers only exposes internal state
// (filter registers, counters) to the parity tests; it does not change any layout.
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <functional>
#include <thread>
#include <vector>

#define private public
#include "jmeters/truepeakdsp.h"
#include "jmeters/kmeterdsp.h"
#include "jmeters/stcorrdsp.h"
#include "jmeters/vumeterdsp.h"
#include "jmeters/iec1ppmdsp.h"
#include "jmeters/iec2ppmdsp.h"
#include "jmeters/msppmdsp.h"
#include "ebumeter/ebu_r128_proc.h"
#include "zita-resampler/resampler-table.h"
#undef private

#include "oracle_api.h"

// The spectrum plugin is a pair of "static include" files (src/meters.cc:672-681);
// ref_spectr_tu.cc compiles them untouched behind a types-only LV2 stub and exports
// these five hooks.
extern "C" {
void* refspec_new (double rate, int nchan);
void  refspec_free (void* s);
void  refspec_run (void* s, const float* l, const float* r, uint32_t n, float speed, float reset, float* ports60);
void  refspec_state (void* s, double* z360, float* val30, float* max30);
void  refspec_coeffs (void* s, double* W);
}

using namespace LV2M;

static void par_for (int n, int nthreads, const std::function<void(int, int)>& fn)
{
    if (nthreads <= 1 || n <= 1) { fn (0, n); return; }
    if (nthreads > n) nthreads = n;
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; ++t) {
        int a = (int)((int64_t)n * t / nthreads), b = (int)((int64_t)n * (t + 1) / nthreads);
        th.emplace_back ([=, &fn] { fn (a, b); });
    }
    for (auto& t : th) t.join ();
}

extern "C" {

const char* orc_kind (void) { return "reference"; }
int orc_hw_threads (void) { return (int)std::thread::hardware_concurrency (); }

/* ------------------------------------------------------------------ EBU */
struct EbuB { int n, nchan; std::vector<Ebu_r128_proc*> p; };

void* orc_ebu_create (int n_inst, int nchan, float fsamp)
{
    EbuB* b = new EbuB; b->n = n_inst; b->nchan = nchan;
    for (int i = 0; i < n_inst; ++i) { Ebu_r128_proc* e = new Ebu_r128_proc; e->init (nchan, fsamp); b->p.push_back (e); }
    return b;
}
void orc_ebu_destroy (void* h) { EbuB* b = (EbuB*)h; for (auto e : b->p) delete e; delete b; }
void orc_ebu_integr (void* h, int inst, int cmd)
{
    EbuB* b = (EbuB*)h;
    for (int i = 0; i < b->n; ++i) {
        if (inst >= 0 && i != inst) continue;
        if (cmd == 0) b->p[i]->integr_pause (); else if (cmd == 1) b->p[i]->integr_start (); else b->p[i]->integr_reset ();
    }
}
void orc_ebu_reset (void* h, int inst)
{
    EbuB* b = (EbuB*)h;
    for (int i = 0; i < b->n; ++i) if (inst < 0 || i == inst) b->p[i]->reset ();
}
void orc_ebu_process (void* h, const float* in, size_t stride, int nfram, int nthreads)
{
    EbuB* b = (EbuB*)h;
    par_for (b->n, nthreads, [=] (int a, int e) {
        for (int i = a; i < e; ++i) {
            float* ip[MAXCH];
            for (int c = 0; c < b->nchan; ++c) ip[c] = const_cast<float*> (in + ((size_t)i * b->nchan + c) * stride);
            b->p[i]->process (nfram, ip);
        }
    });
}
void orc_ebu_read (void* h, float* out)
{
    EbuB* b = (EbuB*)h;
    for (int i = 0; i < b->n; ++i) {
        Ebu_r128_proc* e = b->p[i]; float* o = out + 9 * i;
        o[0] = e->loudness_M (); o[1] = e->maxloudn_M (); o[2] = e->loudness_S (); o[3] = e->maxloudn_S ();
        o[4] = e->integrated (); o[5] = e->integ_thr (); o[6] = e->range_min (); o[7] = e->range_max (); o[8] = e->range_thr ();
    }
}
void orc_ebu_hist (void* h, int inst, int* hm, int* hs, int* c4)
{
    Ebu_r128_proc* e = ((EbuB*)h)->p[inst];
    memcpy (hm, e->histogram_M (), 751 * sizeof (int)); memcpy (hs, e->histogram_S (), 751 * sizeof (int));
    c4[0] = e->hist_M_count (); c4[1] = e->hist_S_count (); c4[2] = e->_hist_M._error; c4[3] = e->_hist_S._error;
}
void orc_ebu_hist_calc (const int* hm, int cm, const int* hs, int cs, float* o)
{
    Ebu_r128_hist M, S;
    memcpy (M._histc, hm, 751 * sizeof (int)); M._count = cm;
    memcpy (S._histc, hs, 751 * sizeof (int)); S._count = cs;
    for (int q = 0; q < 5; ++q) o[q] = -200.0f;
    M.calc_integ (o + 0, o + 1);
    S.calc_range (o + 2, o + 3, o + 4);
}
void orc_ebu_coeffs (void* h, float* o)
{
    Ebu_r128_proc* e = ((EbuB*)h)->p[0];
    o[0] = e->_a0; o[1] = e->_a1; o[2] = e->_a2; o[3] = e->_b1; o[4] = e->_b2; o[5] = e->_c3; o[6] = e->_c4;
}
void orc_ebu_state (void* h, int inst, float* z, float* pw, float* frpwr, int* c4)
{
    EbuB* b = (EbuB*)h; Ebu_r128_proc* e = b->p[inst];
    for (int c = 0; c < b->nchan; ++c) { z[4*c] = e->_fst[c]._z1; z[4*c+1] = e->_fst[c]._z2; z[4*c+2] = e->_fst[c]._z3; z[4*c+3] = e->_fst[c]._z4; }
    memcpy (pw, e->_power, 64 * sizeof (float)); *frpwr = e->_frpwr;
    c4[0] = e->_frcnt; c4[1] = e->_wrind; c4[2] = e->_div1; c4[3] = e->_div2;
}

/* ------------------------------------------------------------------ True peak */
struct TpB { int n; std::vector<TruePeakdsp*> p; };
void* orc_tp_create (int n, float fsamp)
{
    TpB* b = new TpB; b->n = n;
    for (int i = 0; i < n; ++i) { TruePeakdsp* t = new TruePeakdsp; t->init (fsamp); b->p.push_back (t); }
    return b;
}
void orc_tp_destroy (void* h) { TpB* b = (TpB*)h; for (auto t : b->p) delete t; delete b; }
void orc_tp_process (void* h, const float* in, size_t stride, int nfram, int mode, int nthreads)
{
    TpB* b = (TpB*)h;
    par_for (b->n, nthreads, [=] (int a, int e) {
        for (int i = a; i < e; ++i) {
            float* p = const_cast<float*> (in + (size_t)i * stride);
            if (mode) b->p[i]->process_max (p, nfram); else b->p[i]->process (p, nfram);
        }
    });
}
void orc_tp_read (void* h, float* m, float* p) { TpB* b = (TpB*)h; for (int i = 0; i < b->n; ++i) b->p[i]->read (m[i], p[i]); }
void orc_tp_peek (void* h, float* m, float* p, float* z1, float* z2, int* res)
{
    TpB* b = (TpB*)h;
    for (int i = 0; i < b->n; ++i) { TruePeakdsp* t = b->p[i]; m[i] = t->_m; p[i] = t->_p; z1[i] = t->_z1; z2[i] = t->_z2; res[i] = t->_res; }
}
void orc_tp_reset (void* h, int inst) { TpB* b = (TpB*)h; for (int i = 0; i < b->n; ++i) if (inst < 0 || i == inst) b->p[i]->reset (); }
void orc_tp_coeffs (void* h, float* w4, float* ctab)
{
    TruePeakdsp* t = ((TpB*)h)->p[0];
    w4[0] = t->_w1; w4[1] = t->_w2; w4[2] = t->_w3; w4[3] = t->_g;
    Resampler_table* T = t->_src._table;
    memcpy (ctab, T->_ctab, sizeof (float) * T->_hl * (T->_np + 1));
}
void orc_tp_upsample (float fsamp, const float* in, int n, int block, float* out)
{
    TruePeakdsp t; t.init (fsamp);
    for (int o = 0; o < n; o += block) {
        int k = n - o < block ? n - o : block;
        t._src.inp_count = k; t._src.inp_data = const_cast<float*> (in + o);
        t._src.out_count = 4 * k; t._src.out_data = out + 4 * o;
        t._src.process ();
    }
}

void orc_r128_cycle (void* eh, void* th, const float* in, size_t stride, int nfram, int nblocks, int nthreads)
{
    EbuB* e = (EbuB*)eh; TpB* t = (TpB*)th;
    par_for (e->n, nthreads, [=] (int a, int b) {
        for (int i = a; i < b; ++i)
            for (int blk = 0; blk < nblocks; ++blk) {
                float* l = const_cast<float*> (in + (size_t)(2 * i) * stride + (size_t)blk * nfram);
                float* r = const_cast<float*> (in + (size_t)(2 * i + 1) * stride + (size_t)blk * nfram);
                float* ip[2] = {l, r};
                e->p[i]->process (nfram, ip);
                if (t) { t->p[2 * i]->process_max (l, nfram); t->p[2 * i + 1]->process_max (r, nfram); t->p[2 * i]->read (); t->p[2 * i + 1]->read (); }
            }
    });
}

/* ------------------------------------------------------------------ K-meter */
struct KmB { int n; std::vector<Kmeterdsp*> p; };
void* orc_km_create (int n, float fsamp)
{
    KmB* b = new KmB; b->n = n;
    for (int i = 0; i < n; ++i) { Kmeterdsp* k = new Kmeterdsp; k->init (fsamp); b->p.push_back (k); }
    return b;
}
void orc_km_destroy (void* h) { KmB* b = (KmB*)h; for (auto k : b->p) delete k; delete b; }
void orc_km_process (void* h, const float* in, size_t stride, int nfram, int nthreads)
{
    KmB* b = (KmB*)h;
    par_for (b->n, nthreads, [=] (int a, int e) { for (int i = a; i < e; ++i) b->p[i]->process (const_cast<float*> (in + (size_t)i * stride), nfram); });
}
void orc_km_read (void* h, float* rms, float* peak) { KmB* b = (KmB*)h; for (int i = 0; i < b->n; ++i) b->p[i]->read (rms[i], peak[i]); }
void orc_km_peek (void* h, float* s)
{
    KmB* b = (KmB*)h;
    for (int i = 0; i < b->n; ++i) {
        Kmeterdsp* k = b->p[i]; float* o = s + 8 * i;
        o[0] = k->_z1; o[1] = k->_z2; o[2] = k->_rms; o[3] = k->_peak; o[4] = k->_fall; o[5] = (float)k->_cnt; o[6] = (float)k->_fpp; o[7] = k->_flag;
    }
}
void orc_km_reset (void* h, int inst) { KmB* b = (KmB*)h; for (int i = 0; i < b->n; ++i) if (inst < 0 || i == inst) b->p[i]->reset (); }
void orc_km_coeffs (void*, float* omega, int* hold) { *omega = Kmeterdsp::_omega; *hold = Kmeterdsp::_hold; }

/* ------------------------------------------------------------------ needle-meter ballistics */
struct PpmB { int n, kind; std::vector<Vumeterdsp*> vu; std::vector<Iec1ppmdsp*> p1; std::vector<Iec2ppmdsp*> p2; std::vector<Msppmdsp*> ms; };
void* orc_ppm_create (int n, float fsamp, int kind)
{
    PpmB* b = new PpmB; b->n = n; b->kind = kind;
    for (int i = 0; i < n; ++i) {
        if (kind == 0) { b->vu.push_back (new Vumeterdsp); }
        else if (kind == 1) { b->p1.push_back (new Iec1ppmdsp); }
        else if (kind == 2) { b->p2.push_back (new Iec2ppmdsp); }
        else { b->ms.push_back (new Msppmdsp (-6)); b->ms.push_back (new Msppmdsp (-6)); }    /* src/meters.cc:210-212 */
    }
    if (kind == 0) Vumeterdsp::init (fsamp); else if (kind == 1) Iec1ppmdsp::init (fsamp); else if (kind == 2) Iec2ppmdsp::init (fsamp); else Msppmdsp::init (fsamp);
    return b;
}
void orc_ppm_destroy (void* h)
{
    PpmB* b = (PpmB*)h;
    for (auto p : b->vu) delete p; for (auto p : b->p1) delete p; for (auto p : b->p2) delete p; for (auto p : b->ms) delete p;
    delete b;
}
void orc_ppm_process (void* h, const float* in, size_t stride, int nfram, int nthreads)
{
    PpmB* b = (PpmB*)h;
    par_for (b->n, nthreads, [=] (int a, int e) {
        for (int i = a; i < e; ++i) {
            float* p = const_cast<float*> (in + (size_t)i * stride);
            if (b->kind == 0) b->vu[i]->process (p, nfram);
            else if (b->kind == 1) b->p1[i]->process (p, nfram);
            else if (b->kind == 2) b->p2[i]->process (p, nfram);
            else {
                float* l = const_cast<float*> (in + (size_t)(2 * i) * stride); float* r = l + stride;
                b->ms[2 * i]->processM (l, r, nfram); b->ms[2 * i + 1]->processS (l, r, nfram);
            }
        }
    });
}
void orc_ppm_read (void* h, float* out)
{
    PpmB* b = (PpmB*)h;
    for (int i = 0; i < b->n; ++i) {
        if (b->kind == 0) out[i] = b->vu[i]->read (); else if (b->kind == 1) out[i] = b->p1[i]->read (); else if (b->kind == 2) out[i] = b->p2[i]->read ();
        else { out[2 * i] = b->ms[2 * i]->read (); out[2 * i + 1] = b->ms[2 * i + 1]->read (); }
    }
}
void orc_ppm_peek (void* h, float* s)
{
    PpmB* b = (PpmB*)h;
    const int nm = b->kind == 3 ? 2 * b->n : b->n;
    for (int i = 0; i < nm; ++i) {
        float* o = s + 4 * i;
        if (b->kind == 0) { o[0] = b->vu[i]->_z1; o[1] = b->vu[i]->_z2; o[2] = b->vu[i]->_m; o[3] = b->vu[i]->_res; }
        else if (b->kind == 1) { o[0] = b->p1[i]->_z1; o[1] = b->p1[i]->_z2; o[2] = b->p1[i]->_m; o[3] = b->p1[i]->_res; }
        else if (b->kind == 2) { o[0] = b->p2[i]->_z1; o[1] = b->p2[i]->_z2; o[2] = b->p2[i]->_m; o[3] = b->p2[i]->_res; }
        else { o[0] = b->ms[i]->_z1; o[1] = b->ms[i]->_z2; o[2] = b->ms[i]->_m; o[3] = b->ms[i]->_res; }
    }
}
void orc_ppm_set_gain (void* h, float db_m, float db_s)
{
    PpmB* b = (PpmB*)h;
    for (int i = 0; i < (int)b->ms.size () / 2; ++i) { b->ms[2 * i]->set_gain (db_m); b->ms[2 * i + 1]->set_gain (db_s); }
}
void orc_ppm_coeffs (void* h, float* w)
{
    PpmB* b = (PpmB*)h;
    if (b->kind == 0) { w[0] = Vumeterdsp::_w; w[1] = 0; w[2] = 0; w[3] = Vumeterdsp::_g; }
    else if (b->kind == 1) { w[0] = Iec1ppmdsp::_w1; w[1] = Iec1ppmdsp::_w2; w[2] = Iec1ppmdsp::_w3; w[3] = Iec1ppmdsp::_g; }
    else if (b->kind == 2) { w[0] = Iec2ppmdsp::_w1; w[1] = Iec2ppmdsp::_w2; w[2] = Iec2ppmdsp::_w3; w[3] = Iec2ppmdsp::_g; }
    else { w[0] = Msppmdsp::_w1; w[1] = Msppmdsp::_w2; w[2] = Msppmdsp::_w3; w[3] = Msppmdsp::_g; }
}

/* ------------------------------------------------------------------ Stcorr */
struct CorB { int n; std::vector<Stcorrdsp*> p; };
void* orc_cor_create (int n, int fsamp, float flp, float tcf)
{
    CorB* b = new CorB; b->n = n;
    for (int i = 0; i < n; ++i) { Stcorrdsp* c = new Stcorrdsp; c->init (fsamp, flp, tcf); b->p.push_back (c); }
    return b;
}
void orc_cor_destroy (void* h) { CorB* b = (CorB*)h; for (auto c : b->p) delete c; delete b; }
void orc_cor_process (void* h, const float* in, size_t stride, int nfram, int nthreads)
{
    CorB* b = (CorB*)h;
    par_for (b->n, nthreads, [=] (int a, int e) {
        for (int i = a; i < e; ++i)
            b->p[i]->process (const_cast<float*> (in + (size_t)(2 * i) * stride), const_cast<float*> (in + (size_t)(2 * i + 1) * stride), nfram);
    });
}
void orc_cor_read (void* h, float* out) { CorB* b = (CorB*)h; for (int i = 0; i < b->n; ++i) out[i] = b->p[i]->read (); }
void orc_cor_peek (void* h, float* s)
{
    CorB* b = (CorB*)h;
    for (int i = 0; i < b->n; ++i) { Stcorrdsp* c = b->p[i]; float* o = s + 5 * i; o[0] = c->_zl; o[1] = c->_zr; o[2] = c->_zlr; o[3] = c->_zll; o[4] = c->_zrr; }
}
void orc_cor_coeffs (void*, float* w2) { w2[0] = Stcorrdsp::_w1; w2[1] = Stcorrdsp::_w2; }

/* ------------------------------------------------------------------ spectr30 */
struct SpB { int n, nchan; std::vector<void*> p; std::vector<float> ports; };
void* orc_spec_create (int n_inst, int nchan, double rate)
{
    SpB* b = new SpB; b->n = n_inst; b->nchan = nchan; b->ports.assign ((size_t)n_inst * 60, 0.f);
    for (int i = 0; i < n_inst; ++i) { void* s = refspec_new (rate, nchan); if (!s) { delete b; return 0; } b->p.push_back (s); }
    return b;
}
void orc_spec_destroy (void* h) { SpB* b = (SpB*)h; for (auto s : b->p) refspec_free (s); delete b; }
void orc_spec_process (void* h, const float* in, size_t stride, int nfram, float speed, float reset, int nthreads)
{
    SpB* b = (SpB*)h;
    par_for (b->n, nthreads, [=] (int a, int e) {
        for (int i = a; i < e; ++i) {
            const float* l = in + (size_t)i * b->nchan * stride;
            const float* r = b->nchan == 2 ? l + stride : l;
            refspec_run (b->p[i], l, r, (uint32_t)nfram, speed, reset, &b->ports[(size_t)i * 60]);
        }
    });
}
void orc_spec_read (void* h, float* out) { SpB* b = (SpB*)h; memcpy (out, b->ports.data (), b->ports.size () * sizeof (float)); }
void orc_spec_state (void* h, int inst, double* z, float* v, float* m) { refspec_state (((SpB*)h)->p[inst], z, v, m); }
void orc_spec_coeffs (void* h, double* W) { refspec_coeffs (((SpB*)h)->p[0], W); }

/* ------------------------------------------------------------------ bit-meter / SigDistHist through LV2 run() */
void* refplug_new (const char* uri_suffix, double rate);
void  refplug_free (void*);
void  refplug_connect (void*, uint32_t port, void* data);
void  refplug_run (void*, uint32_t n);
void  refbim_mode (void*, int average, int integrating);
void  refbim_snapshot (void*, int32_t*, int32_t*, float*, int64_t*);
void  refsdh_integrate (void*, int on);
void  refsdh_snapshot (void*, int32_t*, int32_t*, double*, int64_t*);

struct PlugB { int n; std::vector<void*> p; };
static void* plug_create (int n, const char* uri, double rate)
{
    PlugB* b = new PlugB; b->n = n;
    for (int i = 0; i < n; ++i) { void* p = refplug_new (uri, rate); if (!p) { delete b; return 0; } b->p.push_back (p); }
    return b;
}
static void plug_process (void* h, const float* in, size_t stride, int nfram, int nthreads)
{
    PlugB* b = (PlugB*)h;
    par_for (b->n, nthreads, [=] (int a, int e) {
        for (int i = a; i < e; ++i) {
            float* p = const_cast<float*> (in + (size_t)i * stride);
            refplug_connect (b->p[i], 2, p); refplug_connect (b->p[i], 3, p);      /* in-place */
            refplug_run (b->p[i], (uint32_t)nfram);
        }
    });
}
void  refebu_ctl (void*, int integrate, int dbtp);
void  refebu_snapshot (void*, float*);
void* orc_ebuplug_create (int n, float rate, int dbtp)
{
    PlugB* b = (PlugB*)plug_create (n, "EBUr128", rate);
    if (b) for (auto p : b->p) refebu_ctl (p, 1, dbtp);
    return b;
}
void  orc_ebuplug_run (void* h, const float* in, size_t stride, int nfram, int nthreads)
{
    PlugB* b = (PlugB*)h;                         /* EBUr128 ports: 2 inL 3 outL 4 inR 5 outR (src/ebulv2.cc:31-38) */
    par_for (b->n, nthreads, [=] (int a, int e) {
        for (int i = a; i < e; ++i) {
            float* l = const_cast<float*> (in + (size_t)(2 * i) * stride); float* r = l + stride;
            refplug_connect (b->p[i], 2, l); refplug_connect (b->p[i], 3, l); refplug_connect (b->p[i], 4, r); refplug_connect (b->p[i], 5, r);
            refplug_run (b->p[i], (uint32_t)nfram);
        }
    });
}
void  orc_ebuplug_read (void* h, float* out) { PlugB* b = (PlugB*)h; for (int i = 0; i < b->n; ++i) refebu_snapshot (b->p[i], out + 10 * i); }
void* orc_bim_create (int n, float rate) { return plug_create (n, "bitmeter", rate); }
void  orc_bim_destroy (void* h) { PlugB* b = (PlugB*)h; for (auto p : b->p) refplug_free (p); delete b; }
void  orc_bim_mode (void* h, int average, int integrating) { PlugB* b = (PlugB*)h; for (auto p : b->p) refbim_mode (p, average, integrating); }
void  orc_bim_process (void* h, const float* in, size_t stride, int nfram, int nthreads) { plug_process (h, in, stride, nfram, nthreads); }
void  orc_bim_read (void* h, int inst, int32_t* hist, int32_t* cnt5, float* mm, int64_t* it) { refbim_snapshot (((PlugB*)h)->p[inst], hist, cnt5, mm, it); }
void* orc_sdh_create (int n, float rate) { return plug_create (n, "SigDistHist", rate); }
void  orc_sdh_destroy (void* h) { orc_bim_destroy (h); }
void  orc_ebuplug_destroy (void* h) { orc_bim_destroy (h); }
void  orc_sdh_integrate (void* h, int on) { PlugB* b = (PlugB*)h; for (auto p : b->p) refsdh_integrate (p, on); }
void  orc_sdh_process (void* h, const float* in, size_t stride, int nfram, int nthreads) { plug_process (h, in, stride, nfram, nthreads); }
void  orc_sdh_read (void* h, int inst, int32_t* hist, int32_t* mp, double* av, int64_t* it) { refsdh_snapshot (((PlugB*)h)->p[inst], hist, mp, av, it); }

/* ------------------------------------------------------------------ DR-14 / TPnRMS through the reference plugins' run() */
struct Dr14B { int n, nch, dr; std::vector<void*> p; std::vector<float> ports; float follow, button; };   /* 19 port floats per instance */
void* orc_dr14_create (int n, int nch, double rate, int dr_mode)
{
    Dr14B* b = new Dr14B; b->n = n; b->nch = nch; b->dr = dr_mode; b->follow = 0; b->button = 0; b->ports.assign ((size_t)n * 19, 0.f);
    const char* uri = dr_mode ? (nch == 2 ? "dr14stereo" : "dr14mono") : (nch == 2 ? "TPnRMSstereo" : "TPnRMSmono");
    for (int i = 0; i < n; ++i) {
        void* p = refplug_new (uri, rate);             /* port 0 = the harness's empty atom sequence; port 1 is re-connected below */
        if (!p) { delete b; return 0; }
        b->p.push_back (p);
        refplug_connect (p, 1, &b->follow); refplug_connect (p, 2, &b->button);                 /* DR_HOST_TRANSPORT, DR_RESET */
        for (int k : {3, 6, 7, 8, 9, 10, 13, 14, 15, 16, 17, 18}) refplug_connect (p, k, &b->ports[(size_t)i * 19 + k]);
    }
    return b;
}
void  orc_dr14_destroy (void* h) { Dr14B* b = (Dr14B*)h; for (auto p : b->p) refplug_free (p); delete b; }
void  orc_dr14_process (void* h, const float* in, size_t stride, int nfram, int nthreads)
{
    Dr14B* b = (Dr14B*)h;                              /* DRPortIndex (src/dr14.c:27-43): 4 in0 5 out0 11 in1 12 out1 */
    par_for (b->n, nthreads, [=] (int a, int e) {
        for (int i = a; i < e; ++i) {
            float* l = const_cast<float*> (in + (size_t)(i * b->nch) * stride); float* r = const_cast<float*> (in + (size_t)(i * b->nch + b->nch - 1) * stride);
            refplug_connect (b->p[i], 4, l); refplug_connect (b->p[i], 5, l); refplug_connect (b->p[i], 11, r); refplug_connect (b->p[i], 12, r);
            refplug_run (b->p[i], (uint32_t)nfram);
        }
    });
    b->button = 0;
}
/* the plugin samples its reset button at the top of run(): latch it for the next process call (state in between is unobservable) */
void  orc_dr14_reset (void* h) { ((Dr14B*)h)->button = 1; }
void  orc_dr14_read (void* h, float* out)
{
    Dr14B* b = (Dr14B*)h;
    for (int i = 0; i < b->n; ++i) {
        const float* p = &b->ports[(size_t)i * 19]; float* o = out + 12 * i;
        o[0] = p[8]; o[1] = p[15]; o[2] = p[6]; o[3] = p[13]; o[4] = p[7]; o[5] = p[14]; o[6] = p[9]; o[7] = p[16]; o[8] = p[10]; o[9] = p[17]; o[10] = p[18]; o[11] = p[3];
    }
}

/* ------------------------------------------------------------------ phasewheel: FFTW3 absent */
void* orc_pw_create (int, int, double) { return 0; }
void  orc_pw_destroy (void*) {}
void  orc_pw_set_mode (void*, int) {}
int   orc_pw_process (void*, const float*, size_t, int, float, int) { return 0; }
void  orc_pw_read (void*, float*, float*, float*) {}
void  orc_pw_raw (void*, int, float*, float*, float*, float*) {}

} // extern "C"

#include "cpu_bench.inc"
