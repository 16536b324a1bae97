// lv2_shim.cu — per-instance LV2 façade over the batched engine: `lv2_descriptor()` with the reference's URIs,
// port indices and run() semantics, so that an LV2 host can load this library where it loaded meters.so.
//
// Covers the 28 pure control-port plugins (src/meters.cc:745-792 lists all 38 descriptors):
//   VU / BBC / EBU / DIN / NOR mono+stereo (run :298-331), BBCM6 (bbcm_run :552-589),
//   COR (cor_run :511-536), dBTPmono/stereo (dbtp_run :438-508), K12/K14/K20 mono/stereo (kmeter_run :333-418),
//   spectr30mono/stereo (spectrum_run, src/spectrumlv2.c:159-257), surround3..8 (sur_run, src/surmeter.c:115-147);
// the plugins with atom ports live in lv2_ebur128.cu (EBUr128), lv2_stats.cu (SigDistHist, bitmeter) and lv2_dr14.cu
// (dr14mono/stereo, TPnRMSmono/stereo).
// lv2_xfer.cu adds phasewheel and stereoscope (raw-audio forwarding to the GUI + correlation), lv2_gon.cu the goniometer, whose
// GUI reaches into the plugin's C struct through LV2 instance-access (ring buffer, mutex: src/goniometer.h): its instance
// handle points at a struct laid out like the reference's.  All 38 descriptors of the reference are served.  In batched mode
// phasewheel and goniometer instances take slots in the COR plugin's hub (cor_hub_join / cor_hub_cycle below).
// Each LV2 instance owns a bank of one instance; run() is synchronous (host buffers in, ports out), exactly the
// reference's calling convention (robtk/jackwrap.c:531-544).  LV2 core types are restated from the LV2
// specification (the SDK is not installed); the struct layout is the stable public C ABI.
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include "lv2_hub.cuh"

namespace b200m {
const LV2_Descriptor* lv2_ebur128_descriptor ();        // lv2_ebur128.cu
const LV2_Descriptor* lv2_sigdisthist_descriptor ();    // lv2_stats.cu
const LV2_Descriptor* lv2_bitmeter_descriptor ();
const LV2_Descriptor* lv2_dr14_descriptor (uint32_t i);   // lv2_dr14.cu: dr14mono, dr14stereo, TPnRMSmono, TPnRMSstereo
const LV2_Descriptor* lv2_xfer_descriptor (uint32_t i);   // lv2_xfer.cu: phasewheel, stereoscope
const LV2_Descriptor* lv2_goniometer_descriptor ();       // lv2_gon.cu
}

namespace {

using namespace b200m;

enum Kind { K_COR, K_DBTP, K_KMETER, K_SPEC, K_NEEDLE, K_BBCM6, K_SUR };
// port enums: src/meters.cc:59-70 (MTR_*), src/spectrumlv2.c:35-44 (SA_*)
enum { MTR_REFLEVEL = 0, MTR_INPUT0, MTR_OUTPUT0, MTR_LEVEL0, MTR_INPUT1, MTR_OUTPUT1, MTR_LEVEL1, MTR_PEAK0, MTR_PEAK1, MTR_HOLD };
enum { SA_SPEED = 60, SA_RESET = 61, SA_AMP = 62, SA_STATE = 63, SA_INPUT0 = 64, SA_OUTPUT0 = 65, SA_INPUT1 = 66, SA_OUTPUT1 = 67 };


struct Shim {
    Kind kind; uint32_t chn;
    b200m_cor* cor = nullptr; b200m_tpk* tpk = nullptr; b200m_spec* spec = nullptr; b200m_ppm* ppm = nullptr;
    float rlgain = 1.0f;                  // needle meters: reference-level gain (src/meters.cc:243,303-306)
    float* port[68] = {nullptr};          // raw port pointers, indexed as in the reference's enums
    PinnedStage stage;                    // [chn] rows, private banks only
    PinnedStage stage2;                   // surround meters: [8] rows = the 4 correlation pairs
    float p_refl = -9999, peak_max[2] = {0, 0}, peak_hold = 0;   // src/meters.cc:245-251
    struct ShimHub* hub = nullptr; int slot = -1;     // batched mode: a slot of a shared bank instead of a private one
};

// batched mode (lv2_hub.cuh): every plugin of this file.  Per-instance controls are stored per slot at submit and reach the bank
// with the cycle's launch: spectr30's speed / reset (b200m_spec_process_ctl_host), BBCM6's S gain (b200m_ppm_set_gain_inst), a
// surround meter's pair selection (the launch gathers the selected rows into the correlation bank's stage), and in the COR hub the
// hold of a phasewheel whose cycle is skipped (b200m_cor_process_ctl_host).  A vacated or newly joined slot is cleared to a
// freshly instantiated plugin.
constexpr uint8_t SUR_IDLE = 0xff;                        // a correlation pair that meters silence (4th pair of surround3, unconnected)

struct ShimHub : SlotHub {
    b200m_cor* cor = nullptr; b200m_tpk* tpk = nullptr; b200m_spec* spec = nullptr; b200m_ppm* ppm = nullptr;
    std::vector<b200m_tpk_result> tpk_res; std::vector<float> f_res;      // results of the last completed cycle
    std::vector<float> spec_ctl;                          // spectr30: [slot] {port 60, port 61} as last submitted
    std::vector<float> s_gain;                            // BBCM6: [slot] S meter gain (dB) as last submitted
    std::vector<uint8_t> sur_sel;                         // surround: [slot][8] input channel of each pair's L and R row, or SUR_IDLE
    std::vector<uint8_t> cor_run;                         // COR: [slot] 0 = held in the open cycle (its bank state left untouched)
    PinnedStage pairs;                                    // surround: [slots * 8] rows, the correlation bank's input

    ShimHub (const HubKey& k, uint32_t n) : SlotHub (k, n) {}
    ~ShimHub () { b200m_cor_destroy (cor); b200m_tpk_destroy (tpk); b200m_spec_destroy (spec); b200m_ppm_destroy (ppm); pairs.release (); }

    static SlotHub* create (const HubKey& k, uint32_t n)
    {
        ShimHub* h = new (std::nothrow) ShimHub (k, n);
        if (!h) return nullptr;
        const uint32_t rows = n * k.chn;
        int rc = -1;
        switch (k.family) {
        case K_COR: rc = b200m_cor_create (&h->cor, 0, n, (int)k.rate, 2e3f, 0.3f); h->f_res.assign (n, 0.0f); h->cor_run.assign (n, 1); break;
        case K_DBTP: case K_KMETER: rc = b200m_tpk_create (&h->tpk, 0, rows, (float)k.rate, k.tpk_flags); h->tpk_res.assign (rows, b200m_tpk_result{0, 0, 0, 0}); break;
        case K_NEEDLE: rc = b200m_ppm_create (&h->ppm, 0, rows, (float)k.rate, k.ppm_kind); h->f_res.assign (rows, 0.0f); break;
        case K_BBCM6: rc = b200m_ppm_create (&h->ppm, 0, n, (float)k.rate, B200M_PPM_MS); h->f_res.assign (2 * n, 0.0f); h->s_gain.assign (n, -6.0f); break;
        case K_SUR:
            rc = b200m_tpk_create (&h->tpk, 0, rows, (float)k.rate, B200M_TPK_KMETER);
            if (!rc) rc = b200m_cor_create (&h->cor, 0, 4 * n, (int)k.rate, 2e3f, 0.3f);
            if (!rc) { h->pairs.reserve (8 * n); if (!h->pairs.cap) rc = -1; }
            h->tpk_res.assign (rows, b200m_tpk_result{0, 0, 0, 0}); h->f_res.assign (4 * n, 0.0f); h->sur_sel.assign (8 * n, SUR_IDLE);
            break;
        case K_SPEC:
            rc = b200m_spec_create (&h->spec, 0, n, k.chn, k.rate); h->f_res.assign ((size_t)n * 60, -100.0f);
            if (!rc) b200m_spec_results (h->spec, h->f_res.data (), nullptr);        // the ports' initial values
            for (uint32_t i = 0; i < n; ++i) { h->spec_ctl.push_back (1.0f); h->spec_ctl.push_back (-4.0f); }   // spectrum_instantiate (:95-98)
            break;
        }
        if (rc) { delete h; return nullptr; }
        return h;
    }
    int launch_bank (uint32_t n) override
    {
        int rc = -1;
        switch (key.family) {
        case K_COR: {
            // the mask reaches the bank only in cycles where a slot holds; every slot runs again in the next cycle unless held anew
            const bool hold = std::find (cor_run.begin (), cor_run.end (), 0) != cor_run.end ();
            rc = b200m_cor_process_ctl_host (cor, stage.data, B200M_MAX_BLOCK, n, hold ? cor_run.data () : nullptr);
            std::fill (cor_run.begin (), cor_run.end (), 1);
            break;
        }
        case K_DBTP: case K_KMETER:
            rc = b200m_tpk_process_host (tpk, stage.data, B200M_MAX_BLOCK, n, B200M_TP_MODE_PROCESS);
            if (!rc) rc = b200m_tpk_read_device (tpk, nullptr);
            break;
        case K_BBCM6:
            for (uint32_t i = 0; i < slots; ++i) b200m_ppm_set_gain_inst (ppm, (int32_t)i, -6, s_gain[i]);     // bbcm_run (src/meters.cc:557-560)
            /* fall through */
        case K_NEEDLE:
            rc = b200m_ppm_process_host (ppm, stage.data, B200M_MAX_BLOCK, n);
            if (!rc) rc = b200m_ppm_read_device (ppm, nullptr);
            break;
        case K_SUR:
            // the selected input rows of every slot -> its 4 correlation pairs; rows of members that skipped the cycle are zero already
            for (uint32_t i = 0; i < slots; ++i)
                for (uint32_t r = 0; r < 8; ++r) {
                    float* dst = pairs.data + (size_t)(8 * i + r) * B200M_MAX_BLOCK;
                    const uint8_t c = sur_sel[8 * i + r];
                    if (c == SUR_IDLE) memset (dst, 0, n * sizeof (float));
                    else memcpy (dst, stage.data + (size_t)(i * key.chn + c) * B200M_MAX_BLOCK, n * sizeof (float));
                }
            rc = b200m_cor_process_host (cor, pairs.data, B200M_MAX_BLOCK, n);
            if (!rc) rc = b200m_tpk_process_host (tpk, stage.data, B200M_MAX_BLOCK, n, B200M_TP_MODE_PROCESS);
            if (!rc) rc = b200m_tpk_read_device (tpk, nullptr);
            break;
        case K_SPEC: rc = b200m_spec_process_ctl_host (spec, stage.data, B200M_MAX_BLOCK, n, spec_ctl.data ()); break;
        }
        return rc;
    }
    void collect () override
    {
        switch (key.family) {
        case K_COR: b200m_cor_results (cor, f_res.data (), nullptr); break;
        case K_DBTP: case K_KMETER: b200m_tpk_results (tpk, tpk_res.data (), nullptr); break;
        case K_NEEDLE: case K_BBCM6: b200m_ppm_results (ppm, f_res.data (), nullptr); break;
        case K_SUR: b200m_cor_results (cor, f_res.data (), nullptr); b200m_tpk_results (tpk, tpk_res.data (), nullptr); break;
        case K_SPEC: b200m_spec_results (spec, f_res.data (), nullptr); break;
        }
    }
    // the slot as a freshly instantiated plugin has it; also at join, because a vacant slot meters silence until it is taken
    void clear (uint32_t slot)
    {
        if (tpk) for (uint32_t c = 0; c < key.chn; ++c) b200m_tpk_clear (tpk, (int32_t)(slot * key.chn + c), nullptr);
        const uint32_t pairs_per_slot = key.family == K_SUR ? 4 : 1;
        if (cor) for (uint32_t c = 0; c < pairs_per_slot; ++c) b200m_cor_clear (cor, (int32_t)(slot * pairs_per_slot + c), nullptr);
        if (ppm) {
            if (key.family == K_BBCM6) { b200m_ppm_clear (ppm, (int32_t)slot, nullptr); s_gain[slot] = -6.0f; }
            else for (uint32_t c = 0; c < key.chn; ++c) b200m_ppm_clear (ppm, (int32_t)(slot * key.chn + c), nullptr);
        }
        if (spec) { b200m_spec_clear (spec, (int32_t)slot, nullptr); spec_ctl[2 * slot] = 1.0f; spec_ctl[2 * slot + 1] = -4.0f; }
        if (!sur_sel.empty ()) memset (&sur_sel[8 * slot], SUR_IDLE, 8);
        if (!cor_run.empty ()) cor_run[slot] = 1;
    }
    void vacate (uint32_t slot) override { clear (slot); }
};

// a slot in a hub with this key, cleared to a freshly instantiated plugin; NULL when batched mode is off
ShimHub* shub_join (const HubKey& key, void* who, int* slot)
{
    ShimHub* hub = (ShimHub*)SlotHub::join (key, who, slot, ShimHub::create);
    if (hub) { std::lock_guard<std::mutex> lh (hub->mu); hub->clear ((uint32_t)*slot); }
    return hub;
}

// one cycle of a batched instance: collect the previous cycle's results of this slot, store its controls, hand in this cycle's
// audio, launch when complete.  ctl: spectr30 {speed, reset}, BBCM6 {S gain}, surround uint8_t[8] pair rows, COR uint8_t hold
// (NULL: runs); NULL for the others.
void hub_cycle (ShimHub* hub, int slot, Kind kind, const float* const* in, uint32_t n, b200m_tpk_result* tr, float* fr, uint32_t nf,
                const void* ctl)
{
    const uint32_t chn = hub->key.chn;
    std::lock_guard<std::mutex> lh (hub->mu);
    hub->close_if_broken (slot, n);
    if (tr) for (uint32_t c = 0; c < chn; ++c) tr[c] = hub->tpk_res[(size_t)slot * chn + c];
    if (fr) for (uint32_t k = 0; k < nf; ++k) fr[k] = hub->f_res[(size_t)slot * nf + k];
    // before a launch by this submit; a member that misses a cycle keeps its previous controls
    if (kind == K_SPEC) memcpy (&hub->spec_ctl[2 * slot], ctl, 2 * sizeof (float));
    else if (kind == K_BBCM6) hub->s_gain[slot] = *(const float*)ctl;
    else if (kind == K_SUR) memcpy (&hub->sur_sel[8 * slot], ctl, 8);
    else if (kind == K_COR && ctl) hub->cor_run[slot] = !*(const uint8_t*)ctl;
    hub->submit (slot, in, n);
}

void shub_cycle (Shim* s, const float* const* in, uint32_t n, b200m_tpk_result* tr, float* fr, uint32_t nf, const void* ctl = nullptr)
{
    hub_cycle (s->hub, s->slot, s->kind, in, n, tr, fr, nf, ctl);
}

LV2_Handle shim_instantiate (const LV2_Descriptor* d, double rate, const char*, const LV2_Feature* const*)
{
    Shim* s = new (std::nothrow) Shim;
    if (!s) return nullptr;
    const char* u = d->URI + strlen (MTR_URI);
    uint32_t tpk_flags = 0; int ppm_kind = 0; bool known = true;
    if (!strcmp (u, "COR")) { s->kind = K_COR; s->chn = 2; }                                                   // :204-207
    else if (!strncmp (u, "dBTP", 4)) { s->kind = K_DBTP; s->chn = strstr (u, "stereo") ? 2 : 1; tpk_flags = B200M_TPK_TRUEPEAK; }
    else if (u[0] == 'K') { s->kind = K_KMETER; s->chn = strstr (u, "stereo") ? 2 : 1; tpk_flags = B200M_TPK_KMETER; }
    else if (!strcmp (u, "BBCM6")) { s->kind = K_BBCM6; s->chn = 2; }               // :208-214
    else if (!strncmp (u, "VU", 2) || !strncmp (u, "BBC", 3) || !strncmp (u, "EBU", 3) || !strncmp (u, "DIN", 3) || !strncmp (u, "NOR", 3)) {
        // MTRDEF (src/meters.cc:172-190,215-219): VU -> Vumeterdsp, BBC/EBU -> Iec2ppmdsp, DIN/NOR -> Iec1ppmdsp
        s->kind = K_NEEDLE; s->chn = strstr (u, "stereo") ? 2 : 1;
        ppm_kind = !strncmp (u, "VU", 2) ? B200M_PPM_VU : (!strncmp (u, "DIN", 3) || !strncmp (u, "NOR", 3)) ? B200M_PPM_IEC1 : B200M_PPM_IEC2;
    }
    else if (!strncmp (u, "surround", 8) && u[8] >= '3' && u[8] <= '8' && !u[9]) { s->kind = K_SUR; s->chn = (uint32_t)(u[8] - '0'); tpk_flags = B200M_TPK_KMETER; }   // src/surmeter.c:24-70
    else if (!strncmp (u, "spectr30", 8)) { s->kind = K_SPEC; s->chn = strstr (u, "stereo") ? 2 : 1; }
    else known = false;
    int rc = known ? 0 : -1;
    if (known) s->hub = shub_join (HubKey{s->kind, ppm_kind, s->chn, tpk_flags, rate}, s, &s->slot);
    if (known && !s->hub) {                                    // a private bank of one instance unless batched mode puts it into a shared one
        switch (s->kind) {
        case K_COR: rc = b200m_cor_create (&s->cor, 0, 1, (int)rate, 2e3f, 0.3f); break;
        case K_DBTP: case K_KMETER: rc = b200m_tpk_create (&s->tpk, 0, s->chn, (float)rate, tpk_flags); break;
        case K_BBCM6: rc = b200m_ppm_create (&s->ppm, 0, 1, (float)rate, B200M_PPM_MS); break;
        case K_NEEDLE: rc = b200m_ppm_create (&s->ppm, 0, s->chn, (float)rate, ppm_kind); break;
        case K_SUR:
            rc = b200m_tpk_create (&s->tpk, 0, s->chn, (float)rate, B200M_TPK_KMETER);
            if (!rc) rc = b200m_cor_create (&s->cor, 0, 4, (int)rate, 2e3f, 0.3f);
            if (rc) { b200m_tpk_destroy (s->tpk); b200m_cor_destroy (s->cor); }
            break;
        case K_SPEC: rc = b200m_spec_create (&s->spec, 0, 1, s->chn, rate); break;
        }
        if (!rc) s->stage.reserve (s->chn);
        if (!rc && s->kind == K_SUR) s->stage2.reserve (8);
    }
    if (rc) { delete s; return nullptr; }                  // instantiate() -> NULL, as the reference does on failure
    return s;
}

void shim_connect (LV2_Handle h, uint32_t port, void* data)
{
    Shim* s = (Shim*)h;
    if (port < 68) s->port[port] = (float*)data;
}

void shim_cleanup (LV2_Handle h)
{
    Shim* s = (Shim*)h;
    if (s->hub) s->hub->leave (s->slot);
    b200m_cor_destroy (s->cor); b200m_tpk_destroy (s->tpk); b200m_spec_destroy (s->spec); b200m_ppm_destroy (s->ppm);
    s->stage.release (); s->stage2.release ();
    delete s;
}

const void* shim_extension_data (const char*) { return nullptr; }

void run_cor (Shim* s, uint32_t off, uint32_t n)
{
    float* in[2] = {s->port[MTR_INPUT0] + off, s->port[MTR_INPUT1] + off};
    float v = 0;
    if (s->hub) { shub_cycle (s, in, n, nullptr, &v, 1); *s->port[MTR_LEVEL0] = v; return; }
    if (!s->stage.fill (in, s->chn, n)) return;
    if (b200m_cor_process_host (s->cor, s->stage.data, s->stage.cap, n) == 0 && b200m_cor_results (s->cor, &v, nullptr) == 0)
        *s->port[MTR_LEVEL0] = v;                          // *level[0] = cor->read() (:516-517)
}

// the "re-use port 0 to request/notify UI" handshake shared by dbtp_run (:444-463) and kmeter_run (:339-357)
bool refl_handshake (Shim* s, bool kmeter)
{
    bool reinit = false;
    const float r = *s->port[MTR_REFLEVEL];
    if (s->p_refl != r) {
        if (fabsf (r) < 3) {
            reinit = true;
            if (kmeter) s->peak_hold = 0; else { s->peak_max[0] = 0; s->peak_max[1] = 0; }
            if (s->hub) { std::lock_guard<std::mutex> lh (s->hub->mu); for (uint32_t c = 0; c < s->chn; ++c) b200m_tpk_reset (s->hub->tpk, (int32_t)(s->slot * s->chn + c), nullptr); }
            else b200m_tpk_reset (s->tpk, -1, nullptr);
        }
        if (kmeter) { if (fabsf (r) == 3) reinit = true; else s->p_refl = r; }
        else if (fabsf (r) != 3) s->p_refl = r;
    }
    if (!kmeter && fabsf (r) == 3) reinit = true;
    return reinit;
}

void run_tpk (Shim* s, uint32_t off, uint32_t n)
{
    const bool km = s->kind == K_KMETER;
    const bool reinit = refl_handshake (s, km);
    // a mono meter re-uses the second channel's port slots for its peak values: only chn audio pointers exist
    float* in[2] = {s->port[MTR_INPUT0] + off, s->chn == 2 ? s->port[MTR_INPUT1] + off : nullptr};
    b200m_tpk_result r[2];
    if (s->hub) shub_cycle (s, in, n, r, nullptr, 0);
    else if (!s->stage.fill (in, s->chn, n) || b200m_tpk_process_host (s->tpk, s->stage.data, s->stage.cap, n, B200M_TP_MODE_PROCESS)) return;
    if (reinit) {                                          // force parameter change (:381-389, :476-489); no read() in such a cycle
        b200m_tpk_result sync[2];
        if (!s->hub) b200m_tpk_results (s->tpk, sync, nullptr);   // stream sync only: run() must not return while the upload of `stage` is in flight
        if (km) { if (s->chn == 1) *s->port[MTR_OUTPUT1] = -1 - (rand () & 0xffff); else *s->port[MTR_HOLD] = -1 - (rand () & 0xffff); }
        else if (s->chn == 1) { *s->port[MTR_LEVEL0] = -500 - (rand () & 0xffff); *s->port[MTR_INPUT1] = -500 - (rand () & 0xffff); }
        else { for (int p : {MTR_LEVEL0, MTR_LEVEL1, MTR_PEAK0, MTR_PEAK1}) *s->port[p] = -500 - (rand () & 0xffff); }
        return;
    }
    if (!s->hub && (b200m_tpk_read_device (s->tpk, nullptr) || b200m_tpk_results (s->tpk, r, nullptr))) return;
    const float rlgain = 1.0f;                             // :243
    if (km) {                                              // :391-407
        if (s->chn == 1) {
            *s->port[MTR_LEVEL0] = rlgain * r[0].km_rms;
            *s->port[MTR_INPUT1] = rlgain * r[0].km_peak;
            if (*s->port[MTR_INPUT1] > s->peak_hold) s->peak_hold = *s->port[MTR_INPUT1];
            *s->port[MTR_OUTPUT1] = s->peak_hold;
        } else {
            for (int c = 0; c < 2; ++c) {
                *s->port[c ? MTR_LEVEL1 : MTR_LEVEL0] = rlgain * r[c].km_rms;
                float* pk = s->port[c ? MTR_PEAK1 : MTR_PEAK0];
                *pk = rlgain * r[c].km_peak;
                if (*pk > s->peak_hold) s->peak_hold = *pk;
            }
            *s->port[MTR_HOLD] = s->peak_hold;
        }
    } else {                                               // :491-507
        for (uint32_t c = 0; c < s->chn; ++c) {
            if (s->peak_max[c] < rlgain * r[c].tp_p) s->peak_max[c] = rlgain * r[c].tp_p;
            *s->port[c ? MTR_LEVEL1 : MTR_LEVEL0] = rlgain * r[c].tp_m;
        }
        if (s->chn == 1) *s->port[MTR_INPUT1] = s->peak_max[0];
        else { *s->port[MTR_PEAK0] = s->peak_max[0]; *s->port[MTR_PEAK1] = s->peak_max[1]; }
    }
}

// run() and bbcm_run() of the needle meters (src/meters.cc:298-331,552-589)
void run_needle (Shim* s, uint32_t off, uint32_t n)
{
    const float r = *s->port[MTR_REFLEVEL];
    if (s->p_refl != r) { s->p_refl = r; s->rlgain = powf (10.0f, 0.05f * (s->p_refl + 18.0)); }
    float* in[2] = {s->port[MTR_INPUT0] + off, s->chn == 2 ? s->port[MTR_INPUT1] + off : nullptr};
    float s_gain = -6;
    if (s->kind == K_BBCM6) {
        const bool s20 = (*s->port[MTR_PEAK0] > 0.5) ? true : false;           // port 7
        s_gain = s20 ? +14 : -6;
        if (!s->hub) b200m_ppm_set_gain (s->ppm, -6, s_gain);
    }
    float v[2] = {0, 0};
    if (s->hub) shub_cycle (s, in, n, nullptr, v, s->chn, &s_gain);
    else if (!s->stage.fill (in, s->chn, n) || b200m_ppm_process_host (s->ppm, s->stage.data, s->stage.cap, n) || b200m_ppm_read_device (s->ppm, nullptr) ||
             b200m_ppm_results (s->ppm, v, nullptr)) return;
    *s->port[MTR_LEVEL0] = s->rlgain * v[0];
    if (s->chn == 2) *s->port[MTR_LEVEL1] = s->rlgain * v[1];
}

void run_spec (Shim* s, uint32_t off, uint32_t n)
{
    float* in[2] = {s->port[SA_INPUT0] + off, s->chn == 2 ? s->port[SA_INPUT1] + off : nullptr};
    float ports[60];
    const float ctl[2] = {*s->port[SA_SPEED], *s->port[SA_RESET]};
    if (s->hub) shub_cycle (s, in, n, nullptr, ports, 60, ctl);
    else if (!s->stage.fill (in, s->chn, n) || b200m_spec_process_host (s->spec, s->stage.data, s->stage.cap, n, *s->port[SA_SPEED], *s->port[SA_RESET]) ||
             b200m_spec_results (s->spec, ports, nullptr)) return;
    for (int i = 0; i < 30; ++i) {
        if (s->port[i]) *s->port[i] = ports[i];
        if (s->port[30 + i]) *s->port[30 + i] = ports[30 + i] <= -500.0f ? -500.0f - (rand () & 0xffff) : ports[30 + i];   // :243-246
    }
}

// sur_run (src/surmeter.c:115-147): 3 or 4 selectable-pair correlation meters + one K-meter per channel
void run_sur (Shim* s, uint32_t off, uint32_t n)
{
    float* in[8];
    for (uint32_t c = 0; c < s->chn; ++c) { in[c] = s->port[13 + 4 * c]; if (!in[c]) return; in[c] += off; }
    const uint32_t cors = s->chn > 3 ? 4 : 3;
    uint8_t sel[8];                                        // SUR_IDLE rows stage silence: cor4[3] idles on a 3-channel meter
    memset (sel, SUR_IDLE, sizeof (sel));
    for (uint32_t c = 0; c < cors; ++c) {
        if (!s->port[1 + 3 * c] || !s->port[2 + 3 * c]) continue;
        uint32_t in_a = (uint32_t)rintf (*s->port[1 + 3 * c]), in_b = (uint32_t)rintf (*s->port[2 + 3 * c]);
        if (in_a >= s->chn) in_a = s->chn - 1;
        if (in_b >= s->chn) in_b = s->chn - 1;
        sel[2 * c] = (uint8_t)in_a; sel[2 * c + 1] = (uint8_t)in_b;
    }
    float cv[4] = {0, 0, 0, 0};
    b200m_tpk_result r[8];
    if (s->hub) shub_cycle (s, in, n, r, cv, 4, sel);
    else {
        const float* pair[8];
        for (int k = 0; k < 8; ++k) pair[k] = sel[k] == SUR_IDLE ? nullptr : in[sel[k]];
        if (!s->stage2.fill (pair, 8, n) || b200m_cor_process_host (s->cor, s->stage2.data, s->stage2.cap, n) || b200m_cor_results (s->cor, cv, nullptr)) return;
    }
    for (uint32_t c = 0; c < cors; ++c) if (s->port[3 + 3 * c]) *s->port[3 + 3 * c] = cv[c];
    if (!s->hub && (!s->stage.fill (in, s->chn, n) || b200m_tpk_process_host (s->tpk, s->stage.data, s->stage.cap, n, B200M_TP_MODE_PROCESS) ||
                    b200m_tpk_read_device (s->tpk, nullptr) || b200m_tpk_results (s->tpk, r, nullptr))) return;
    for (uint32_t c = 0; c < s->chn; ++c) {
        if (s->port[15 + 4 * c]) *s->port[15 + 4 * c] = r[c].km_rms;         // Kmeterdsp::read (m, p): *level = m, *peak = p
        if (s->port[16 + 4 * c]) *s->port[16 + 4 * c] = r[c].km_peak;
    }
}

void shim_run (LV2_Handle h, uint32_t n)
{
    Shim* s = (Shim*)h;
    if (n == 0) return;
    // Audio is forwarded FIRST and unconditionally (every reference run() ends in the in -> out memcpy, src/meters.cc:326-330,
    // :415-417, :531-535; src/spectrumlv2.c:249-256; src/surmeter.c:143-146): a metering failure -- no memory, a CUDA error --
    // may cost a meter reading, never the audio.  run() itself never fails (SURVEY §8b).
    {
        float* in[8] = {nullptr}; float* out[8] = {nullptr};
        if (s->kind == K_SUR) for (uint32_t c = 0; c < s->chn; ++c) { in[c] = s->port[13 + 4 * c]; out[c] = s->port[14 + 4 * c]; }
        else if (s->kind == K_SPEC) { in[0] = s->port[SA_INPUT0]; out[0] = s->port[SA_OUTPUT0]; if (s->chn == 2) { in[1] = s->port[SA_INPUT1]; out[1] = s->port[SA_OUTPUT1]; } }
        else { in[0] = s->port[MTR_INPUT0]; out[0] = s->port[MTR_OUTPUT0]; if (s->chn == 2) { in[1] = s->port[MTR_INPUT1]; out[1] = s->port[MTR_OUTPUT1]; } }
        forward_audio (in, out, s->chn, n);
        for (uint32_t c = 0; c < s->chn; ++c) if (!in[c]) return;          // unconnected input: nothing to meter
    }
    // the engine's block limit is 8192 frames (B200M_MAX_BLOCK = the hosts' MAXPERIOD); the reference's needle / COR / K-meter /
    // spectrum plugins take any n, so longer cycles are metered in pieces of at most 8192 frames
    for (uint32_t off = 0; off < n; off += B200M_MAX_BLOCK) {
        const uint32_t k = n - off < B200M_MAX_BLOCK ? n - off : B200M_MAX_BLOCK;
        switch (s->kind) {
        case K_COR: run_cor (s, off, k); break;
        case K_DBTP: case K_KMETER: run_tpk (s, off, k); break;
        case K_SPEC: run_spec (s, off, k); break;
        case K_NEEDLE: case K_BBCM6: run_needle (s, off, k); break;
        case K_SUR: run_sur (s, off, k); break;
        }
    }
}

#define DESC(NAME) {MTR_URI NAME, shim_instantiate, shim_connect, nullptr, shim_run, nullptr, shim_cleanup, shim_extension_data}
const LV2_Descriptor g_desc[] = {
    DESC ("VUmono"), DESC ("VUstereo"), DESC ("BBCmono"), DESC ("BBCstereo"), DESC ("EBUmono"), DESC ("EBUstereo"),
    DESC ("DINmono"), DESC ("DINstereo"), DESC ("NORmono"), DESC ("NORstereo"), DESC ("BBCM6"),
    DESC ("COR"), DESC ("spectr30mono"), DESC ("dBTPmono"), DESC ("dBTPstereo"),
    DESC ("K12mono"), DESC ("K14mono"), DESC ("K20mono"), DESC ("K12stereo"), DESC ("K14stereo"), DESC ("K20stereo"),
    DESC ("spectr30stereo"),
    DESC ("surround8"), DESC ("surround7"), DESC ("surround6"), DESC ("surround5"), DESC ("surround4"), DESC ("surround3"),
};

}  // namespace

namespace b200m {
// phasewheel and goniometer run the COR plugin's Stcorrdsp, init (rate, 2e3f, 0.3f) on two rows (src/xfer.c:93, src/goniometerlv2.c:73-74)
SlotHub* cor_hub_join (double rate, void* who, int* slot) { return shub_join (HubKey{K_COR, 0, 2, 0, rate}, who, slot); }

float cor_hub_cycle (SlotHub* hub, int slot, const float* const* in, uint32_t n, bool hold)
{
    float v = 0;
    const uint8_t h = hold;
    hub_cycle ((ShimHub*)hub, slot, K_COR, in, n, nullptr, &v, 1, &h);
    return v;
}
}

// The one symbol meters.so exports (src/meters.cc:739-792).  Hosts look plugins up by URI; the indices here are
// the covered subset in the reference's order.
extern "C" __attribute__ ((visibility ("default"))) const LV2_Descriptor* lv2_descriptor (uint32_t index)
{
    constexpr uint32_t n = sizeof (g_desc) / sizeof (g_desc[0]);
    if (index < n) return &g_desc[index];
    if (index == n) return b200m::lv2_ebur128_descriptor ();       // the atom-port plugins follow the control-port ones
    if (index == n + 1) return b200m::lv2_sigdisthist_descriptor ();
    if (index == n + 2) return b200m::lv2_bitmeter_descriptor ();
    if (index < n + 7) return b200m::lv2_dr14_descriptor (index - (n + 3));
    if (index < n + 9) return b200m::lv2_xfer_descriptor (index - (n + 7));
    if (index == n + 9) return b200m::lv2_goniometer_descriptor ();
    return nullptr;
}
