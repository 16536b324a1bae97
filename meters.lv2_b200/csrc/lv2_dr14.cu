// lv2_dr14.cu — the dr14mono / dr14stereo / TPnRMSmono / TPnRMSstereo plugins (descriptors 25-28 of the reference,
// src/meters.cc:771-774) over a one-instance b200m_dr14 bank: ports as DRPortIndex (src/dr14.c:27-43), the atom control
// port (time:Position -> reset on transport start, dr14reset, meteron / meteroff), the reset button and the
// "force a GUI update" values of dr14_run (:359-382,464-475).  All metering runs on the GPU (dr14.cu); results appear on
// the float control ports.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "lv2_hub.cuh"

namespace {

using namespace b200m;

enum { DR_CONTROL = 0, DR_HOST_TRANSPORT, DR_RESET, DR_BLKCNT, DR_INPUT0, DR_OUTPUT0, DR_V_PEAK0, DR_M_PEAK0, DR_V_RMS0, DR_M_RMS0, DR_DR0,
       DR_INPUT1, DR_OUTPUT1, DR_V_PEAK1, DR_M_PEAK1, DR_V_RMS1, DR_M_RMS1, DR_DR1, DR_TOTAL, DR_NPORTS };

struct DrPlugin {
    b200m_dr14* bank = nullptr; uint32_t nch = 1; bool dr_mode = false;
    PinnedStage stage;
    void* port[DR_NPORTS] = {nullptr};
    LV2_URID atom_Blank = 0, atom_Object = 0, atom_Float = 0, time_Position = 0, time_speed = 0, dr14reset = 0, meteron = 0, meteroff = 0;
    bool transport_rolling = false, reinit_gui = false;
};

float* fport (DrPlugin* p, int i) { return (float*)p->port[i]; }

LV2_Handle dr_instantiate (const LV2_Descriptor* d, double rate, const char*, const LV2_Feature* const* features)
{
    const char* u = d->URI + strlen (MTR_URI);
    uint32_t nch; bool dr_mode;
    if (!strcmp (u, "dr14stereo")) { nch = 2; dr_mode = true; }
    else if (!strcmp (u, "dr14mono")) { nch = 1; dr_mode = true; }
    else if (!strcmp (u, "TPnRMSstereo")) { nch = 2; dr_mode = false; }
    else if (!strcmp (u, "TPnRMSmono")) { nch = 1; dr_mode = false; }
    else return nullptr;
    const LV2_URID_Map* map = find_urid_map (features);
    if (!map) { fprintf (stderr, "DR14LV2 error: Host does not support urid:map\n"); return nullptr; }      // :133-136
    DrPlugin* p = new (std::nothrow) DrPlugin;
    if (!p) return nullptr;
    p->nch = nch; p->dr_mode = dr_mode;
    auto M = [&] (const char* uri) { return map->map (map->handle, uri); };
    p->atom_Blank = M (B200M_LV2_ATOM "Blank"); p->atom_Object = M (B200M_LV2_ATOM "Object"); p->atom_Float = M (B200M_LV2_ATOM "Float");
    p->time_Position = M (B200M_LV2_TIME "Position"); p->time_speed = M (B200M_LV2_TIME "speed");
    p->dr14reset = M (MTR_URI "dr14reset"); p->meteron = M (MTR_URI "meteron"); p->meteroff = M (MTR_URI "meteroff");
    if (b200m_dr14_create (&p->bank, 0, 1, nch, rate, dr_mode)) { delete p; return nullptr; }
    p->stage.reserve (nch);
    return p;
}

void dr_connect (LV2_Handle h, uint32_t port, void* data) { DrPlugin* p = (DrPlugin*)h; if (port < DR_NPORTS) p->port[port] = data; }

void dr_run (LV2_Handle h, uint32_t n)
{
    DrPlugin* p = (DrPlugin*)h;
    float* in[2] = {fport (p, DR_INPUT0), fport (p, DR_INPUT1)}; float* out[2] = {fport (p, DR_OUTPUT0), fport (p, DR_OUTPUT1)};
    // audio first (dr14_run ends with this copy, src/dr14.c:477-481): no metering failure may drop it.  TruePeakdsp::process
    // itself is limited to 8192 frames (jmeters/truepeakdsp.cc:43-44), so longer cycles are forwarded but not metered.
    forward_audio (in, out, p->nch, n);
    if (!in[0] || (p->nch == 2 && !in[1]) || n < 1 || n > B200M_MAX_BLOCK) return;
    const bool follow_host_transport = fport (p, DR_HOST_TRANSPORT) && *fport (p, DR_HOST_TRANSPORT) != 0;
    bool reset = false;
    if (p->port[DR_CONTROL]) {                                 // events: reset from the GUI, transport from the host (:361-379)
        for (AtomEvents ev (p->port[DR_CONTROL]); ev.valid (); ev.next ()) {
            const AtomHead* a = ev.body ();
            if (a->type != p->atom_Blank && a->type != p->atom_Object) continue;
            AtomObject obj; obj.a = a;
            const uint32_t ot = obj.otype ();
            if (ot == p->time_Position) {                      // parse_time_position (:260-280)
                const AtomHead* speed = obj.get (p->time_speed);
                if (speed && speed->type == p->atom_Float && speed->size >= 4) {
                    const float ts = *(const float*)(speed + 1);
                    if (ts != 0 && !p->transport_rolling && follow_host_transport) reset = true;
                    p->transport_rolling = ts != 0;
                }
            }
            if (ot == p->dr14reset) reset = true;
            if (ot == p->meteron) p->reinit_gui = true;
            if (ot == p->meteroff) p->reinit_gui = false;
        }
    }
    if (fport (p, DR_RESET) && *fport (p, DR_RESET) != 0) reset = true;
    if (reset) b200m_dr14_reset (p->bank, nullptr);           // reset_peaks is idempotent: several triggers in one cycle = one reset

    b200m_dr14_result r;
    if (!p->stage.fill (in, p->nch, n) || b200m_dr14_run_host (p->bank, p->stage.data, p->stage.cap, n) || b200m_dr14_results (p->bank, &r, nullptr)) return;

    static const int pv_peak[2] = {DR_V_PEAK0, DR_V_PEAK1}, pm_peak[2] = {DR_M_PEAK0, DR_M_PEAK1}, pv_rms[2] = {DR_V_RMS0, DR_V_RMS1},
                     pm_rms[2] = {DR_M_RMS0, DR_M_RMS1}, p_dr[2] = {DR_DR0, DR_DR1};
    auto W = [&] (int port, float v) { if (p->port[port]) *fport (p, port) = v; };
    for (uint32_t c = 0; c < p->nch; ++c) {                    // :425-447
        W (pv_rms[c], r.v_rms[c]); W (pv_peak[c], r.v_peak[c]); W (pm_peak[c], r.m_peak[c]); W (pm_rms[c], r.m_rms[c]);
        if (p->dr_mode) W (p_dr[c], r.dr[c]);
    }
    if (p->nch > 1 && p->dr_mode) W (DR_TOTAL, r.dr_total);
    W (DR_BLKCNT, r.block_count);
    if (p->reinit_gui) {                                       // force the GUI to redraw everything (:464-475)
        if (p->nch > 1 && p->dr_mode) W (DR_TOTAL, 21);
        for (uint32_t c = 0; c < p->nch; ++c) { W (pm_peak[c], -100); W (pm_rms[c], -100); if (p->dr_mode) W (p_dr[c], 21); }
        W (DR_BLKCNT, -1 - (rand () & 0xffff));
    }
}

void dr_cleanup (LV2_Handle h)
{
    DrPlugin* p = (DrPlugin*)h;
    b200m_dr14_destroy (p->bank);
    p->stage.release ();
    delete p;
}

const void* dr_extension_data (const char*) { return nullptr; }

#define DRDESC(NAME) {MTR_URI NAME, dr_instantiate, dr_connect, nullptr, dr_run, nullptr, dr_cleanup, dr_extension_data}
const LV2_Descriptor g_dr[4] = {DRDESC ("dr14mono"), DRDESC ("dr14stereo"), DRDESC ("TPnRMSmono"), DRDESC ("TPnRMSstereo")};

}  // namespace

namespace b200m { const LV2_Descriptor* lv2_dr14_descriptor (uint32_t i) { return i < 4 ? &g_dr[i] : nullptr; } }
