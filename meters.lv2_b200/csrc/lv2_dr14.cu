// lv2_dr14.cu — the dr14mono / dr14stereo / TPnRMSmono / TPnRMSstereo plugins (descriptors 25-28 of the reference,
// src/meters.cc:771-774) over a one-instance b200m_dr14 bank: ports as DRPortIndex (src/dr14.c:27-43), the atom control
// port (time:Position -> reset on transport start, dr14reset, meteron / meteroff), the reset button and the
// "force a GUI update" values of dr14_run (:359-382,464-475).  All metering runs on the GPU (dr14.cu); results appear on
// the float control ports.  In batched mode (lv2_hub.cuh) the instances of one sample rate, channel count and mode share one bank
// (DrHub): every slot has its own reset_peaks and 3 s window phase, so a batched instance's ports after cycle k + 1 are a
// private instance's after cycle k.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "lv2_hub.cuh"

namespace {

using namespace b200m;

enum { DR_CONTROL = 0, DR_HOST_TRANSPORT, DR_RESET, DR_BLKCNT, DR_INPUT0, DR_OUTPUT0, DR_V_PEAK0, DR_M_PEAK0, DR_V_RMS0, DR_M_RMS0, DR_DR0,
       DR_INPUT1, DR_OUTPUT1, DR_V_PEAK1, DR_M_PEAK1, DR_V_RMS1, DR_M_RMS1, DR_DR1, DR_TOTAL, DR_NPORTS };

// batched mode: one b200m_dr14 bank per (rate, channels, mode).  Resets recorded in run() k (under mu, after the cycle before it
// was closed) are applied in one b200m_dr14_control call at the launch of cycle k, ahead of its audio, where dr14_run applies
// them.  A slot's next tenant is cleared at the launch of ITS first cycle, so its window phase starts with its first run().
struct DrHub : SlotHub {
    b200m_dr14* bank = nullptr;
    std::vector<b200m_dr14_result> res;                        // the last completed cycle, per slot
    std::vector<uint8_t> fresh;                                // per slot: clear it at the launch of its tenant's first cycle
    std::vector<uint32_t> resets, clears;                      // slots to reset / clear at the next launch

    DrHub (const HubKey& k, uint32_t n) : SlotHub (k, n), res (n), fresh (n, 1) {}
    ~DrHub () { b200m_dr14_destroy (bank); }

    static SlotHub* create (const HubKey& k, uint32_t n)
    {
        DrHub* h = new (std::nothrow) DrHub (k, n);
        if (!h) return nullptr;
        if (b200m_dr14_create (&h->bank, 0, n, k.chn, k.rate, (int)k.tpk_flags)) { delete h; return nullptr; }
        return h;
    }
    // with mu held, after close_if_broken: this run()'s reset (several triggers = one reset_peaks) and a new tenant's clear
    void record (int slot, bool reset)
    {
        if (fresh[slot]) { fresh[slot] = 0; clears.push_back ((uint32_t)slot); }
        else if (reset) resets.push_back ((uint32_t)slot);
    }
    int launch_bank (uint32_t n) override
    {
        int rc = 0;
        if (!clears.empty ()) rc = b200m_dr14_control (bank, clears.data (), (uint32_t)clears.size (), B200M_DR14_CLEAR, nullptr);
        if (!rc && !resets.empty ()) rc = b200m_dr14_control (bank, resets.data (), (uint32_t)resets.size (), B200M_DR14_RESET, nullptr);
        clears.clear (); resets.clear ();
        return rc ? rc : b200m_dr14_run_host (bank, stage.data, B200M_MAX_BLOCK, n);
    }
    void collect () override { b200m_dr14_results (bank, res.data (), nullptr); }
    void vacate (uint32_t slot) override { fresh[slot] = 1; }
};

struct DrPlugin {
    b200m_dr14* bank = nullptr; uint32_t nch = 1; bool dr_mode = false;
    DrHub* hub = nullptr; int slot = -1;
    bool last_valid = false, last_reinit = false;              // batched: the previous cycle was submitted, and its reinit_gui
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
    p->hub = (DrHub*)SlotHub::join (HubKey{HUB_DR14, 0, nch, dr_mode ? 1u : 0u, rate}, p, &p->slot, DrHub::create);
    if (p->hub) return p;
    if (b200m_dr14_create (&p->bank, 0, 1, nch, rate, dr_mode)) { delete p; return nullptr; }
    p->stage.reserve (nch);
    return p;
}

void dr_connect (LV2_Handle h, uint32_t port, void* data) { DrPlugin* p = (DrPlugin*)h; if (port < DR_NPORTS) p->port[port] = data; }

// the port values of one cycle's results (:425-475), with that cycle's reinit_gui
void dr_publish (DrPlugin* p, const b200m_dr14_result& r, bool reinit)
{
    static const int pv_peak[2] = {DR_V_PEAK0, DR_V_PEAK1}, pm_peak[2] = {DR_M_PEAK0, DR_M_PEAK1}, pv_rms[2] = {DR_V_RMS0, DR_V_RMS1},
                     pm_rms[2] = {DR_M_RMS0, DR_M_RMS1}, p_dr[2] = {DR_DR0, DR_DR1};
    auto W = [&] (int port, float v) { if (p->port[port]) *fport (p, port) = v; };
    for (uint32_t c = 0; c < p->nch; ++c) {                    // :425-447
        W (pv_rms[c], r.v_rms[c]); W (pv_peak[c], r.v_peak[c]); W (pm_peak[c], r.m_peak[c]); W (pm_rms[c], r.m_rms[c]);
        if (p->dr_mode) W (p_dr[c], r.dr[c]);
    }
    if (p->nch > 1 && p->dr_mode) W (DR_TOTAL, r.dr_total);
    W (DR_BLKCNT, r.block_count);
    if (reinit) {                                              // force the GUI to redraw everything (:464-475)
        if (p->nch > 1 && p->dr_mode) W (DR_TOTAL, 21);
        for (uint32_t c = 0; c < p->nch; ++c) { W (pm_peak[c], -100); W (pm_rms[c], -100); if (p->dr_mode) W (p_dr[c], 21); }
        W (DR_BLKCNT, -1 - (rand () & 0xffff));
    }
}

void dr_run (LV2_Handle h, uint32_t n)
{
    DrPlugin* p = (DrPlugin*)h;
    float* in[2] = {fport (p, DR_INPUT0), fport (p, DR_INPUT1)}; float* out[2] = {fport (p, DR_OUTPUT0), fport (p, DR_OUTPUT1)};
    // audio first (dr14_run ends with this copy, src/dr14.c:477-481): no metering failure may drop it.  TruePeakdsp::process
    // itself is limited to 8192 frames (jmeters/truepeakdsp.cc:43-44), so longer cycles are forwarded but not metered.
    forward_audio (in, out, p->nch, n);
    if (!in[0] || (p->nch == 2 && !in[1]) || n < 1 || n > B200M_MAX_BLOCK) { p->last_valid = false; return; }
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

    if (p->hub) {                                              // the previous cycle's ports; this cycle's reset lands ahead of its audio
        std::lock_guard<std::mutex> lh (p->hub->mu);
        p->hub->close_if_broken (p->slot, n);
        p->hub->record (p->slot, reset);
        p->hub->submit (p->slot, in, n);
        if (p->last_valid) dr_publish (p, p->hub->res[p->slot], p->last_reinit);
        p->last_valid = true; p->last_reinit = p->reinit_gui;
        return;
    }
    if (reset) b200m_dr14_reset (p->bank, nullptr);           // reset_peaks is idempotent: several triggers in one cycle = one reset
    b200m_dr14_result r;
    if (!p->stage.fill (in, p->nch, n) || b200m_dr14_run_host (p->bank, p->stage.data, p->stage.cap, n) || b200m_dr14_results (p->bank, &r, nullptr)) return;
    dr_publish (p, r, p->reinit_gui);
}

void dr_cleanup (LV2_Handle h)
{
    DrPlugin* p = (DrPlugin*)h;
    if (p->hub) p->hub->leave (p->slot);
    b200m_dr14_destroy (p->bank);
    p->stage.release ();
    delete p;
}

const void* dr_extension_data (const char*) { return nullptr; }

#define DRDESC(NAME) {MTR_URI NAME, dr_instantiate, dr_connect, nullptr, dr_run, nullptr, dr_cleanup, dr_extension_data}
const LV2_Descriptor g_dr[4] = {DRDESC ("dr14mono"), DRDESC ("dr14stereo"), DRDESC ("TPnRMSmono"), DRDESC ("TPnRMSstereo")};

}  // namespace

namespace b200m { const LV2_Descriptor* lv2_dr14_descriptor (uint32_t i) { return i < 4 ? &g_dr[i] : nullptr; } }
