// lv2_ebur128.cu — the EBUr128 plugin (descriptor 11 of the reference, src/meters.cc:759) over a one-instance
// b200m_r128 bank: same URI, ports, control-message protocol, notify-port messages and state extension as
// src/ebulv2.cc, so the reference's own GUI (or any LV2 host) can sit on top of it.
//
//   ports        EBU_CONTROL 0 (atom in), EBU_NOTIFY 1 (atom out), in/out L 2/3, in/out R 4/5          (:31-38)
//   control in   time:Position (transport follow), meteron / meteroff, metercfg {controlkey, controlval} (:258-331)
//   notify out   control {key,val} replies, rdr_radarpoint (resync batch + live), rdr_histpoint / rdr_histogram
//                (histogram deltas, bins 110..649, at most 17 per cycle), ebulevels                     (:250-482)
//   state        one atom:Int "ebu_state" = ui_settings | follow_transport_mode << 8 | radar_spd_max << 16 (:513-548)
//
// The audio cycle (ebu->process, process_max x 2, getters, coef_to_db hold) runs on the GPU through b200m_r128_*;
// everything else in ebur128_run is host-side message bookkeeping, restated here message for message so that the
// bytes in the notify buffer equal the reference's (tests/test_lv2_ebur128_gpu.py compares them).
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "lv2_hub.cuh"

namespace {

using namespace b200m;

enum { EBU_CONTROL = 0, EBU_NOTIFY, EBU_INPUT0, EBU_OUTPUT0, EBU_INPUT1, EBU_OUTPUT1 };
// numeric control keys, src/uris.h:187-203
enum { CTL_START = 1, CTL_PAUSE, CTL_RESET, CTL_TRANSPORTSYNC, CTL_AUTORESET, CTL_RADARTIME, CTL_UISETTINGS,
       CTL_LV2_RADARTIME, CTL_LV2_FTM, CTL_LV2_RESETRADAR, CTL_LV2_RESYNCDONE };
constexpr int HIST_LEN = 751, RADAR_POINTS = 360;

struct Urids {
    LV2_URID atom_Blank, atom_Object, atom_Int, atom_Float, atom_Bool, atom_Sequence;
    LV2_URID time_Position, time_speed;
    LV2_URID control, cckey, ccval, meteron, meteroff, metercfg;
    LV2_URID ebulevels, loudnessM, maxloudnM, loudnessS, maxloudnS, integrated, range_min, range_max, integrating, integr_time, truepeak;
    LV2_URID ebu_state, rdr_histogram, rdr_histpoint, rdr_radarpoint, rdr_pointpos, rdr_pos_cur, rdr_pos_max;
};

struct EbuHub;
struct EbuPlugin {
    b200m_r128* bank = nullptr; EbuHub* hub = nullptr; int slot = -1;       // private bank of one, or slot `slot` of a shared bank
    PinnedStage stage;                                         // private bank only
    Urids u; AtomWriter out;
    const void* control = nullptr; void* notify = nullptr;
    float* input[2] = {nullptr, nullptr}; float* output[2] = {nullptr, nullptr};
    double rate = 48000;
    bool ui_active = false, transport_rolling = false, integrating = false, dbtp_enable = false, send_state_to_ui = false;
    int follow_transport_mode = 0;
    float radarS[RADAR_POINTS], radarM[RADAR_POINTS], radarSC = -INFINITY, radarMC = -INFINITY;
    int radar_pos_cur = 0, radar_pos_max = RADAR_POINTS, radar_resync = -1;
    uint32_t radar_spd_cur = 0, radar_spd_max = 0;
    uint64_t integration_time = 0;
    uint32_t ui_settings = 8;
    int sentM[HIST_LEN], sentS[HIST_LEN], hist_maxM = 0, hist_maxS = 0;   // what the UI has been told so far
    int32_t histM[HIST_LEN], histS[HIST_LEN];
};

// batched mode (lv2_hub.cuh): the instances of one sample rate share one bank.  A slot's tenant gets a fresh instance whose own
// 50 ms fragment clock starts with its first run() (B200M_R128_NEW, applied ahead of that run's control messages and audio).
// Each slot's dBTP switch is its member's own (b200m_r128_set_dbtp_inst at the launch of the cycle): while it is off the slot's
// true-peak histories stay frozen and its hold reads -inf, as the plugin's do.
struct EbuHub : SlotHub {
    b200m_r128* bank = nullptr;
    std::vector<b200m_ebu_result> res; std::vector<float> tp;  // results of the last completed cycle
    std::vector<uint8_t> fresh;                                // per slot: its tenant has not run yet
    std::vector<uint8_t> dbtp;                                 // per slot: the dBTP switch the bank has

    EbuHub (const HubKey& k, uint32_t n) : SlotHub (k, n), res (n), tp (n, -INFINITY), fresh (n, 1), dbtp (n, 0) {}
    ~EbuHub () { b200m_r128_destroy (bank); }

    static SlotHub* create (const HubKey& k, uint32_t n)
    {
        EbuHub* h = new (std::nothrow) EbuHub (k, n);
        if (!h) return nullptr;
        if (b200m_r128_create (&h->bank, 0, n, (float)k.rate, 0)) { delete h; return nullptr; }
        b200m_r128_results (h->bank, h->res.data (), h->tp.data (), nullptr);     // the getters' initial values
        return h;
    }
    int launch_bank (uint32_t n) override
    {
        for (uint32_t s = 0; s < slots; ++s) {                 // a vacant slot keeps its last switch
            const EbuPlugin* m = (const EbuPlugin*)member[s];
            if (m && m->dbtp_enable != (dbtp[s] != 0)) { dbtp[s] = m->dbtp_enable; b200m_r128_set_dbtp_inst (bank, (int32_t)s, m->dbtp_enable); }
        }
        return b200m_r128_run_host (bank, stage.data, B200M_MAX_BLOCK, n);
    }
    void collect () override { b200m_r128_results (bank, res.data (), tp.data (), nullptr); }
    // with mu held, after close_if_broken, before the run()'s control messages: the instance the plugin's constructor made
    // (Ebu_r128_proc::reset, src/ebulv2.cc:190) starts at the cycle this run() joins
    void first_run (int slot)
    {
        if (!fresh[slot]) return;
        fresh[slot] = 0;
        b200m_r128_control (bank, slot, B200M_R128_NEW, nullptr);
    }
    void vacate (uint32_t slot) override
    {
        // the vacated slot idles as a freshly created instance on silence: filters, 64-fragment ring, loudness values, histograms,
        // true-peak history and hold all cleared; its next tenant restarts the fragment clock at its first run()
        fresh[slot] = 1;
        b200m_r128_control (bank, (int)slot, B200M_R128_CLEAR, nullptr);
        tp[slot] = -INFINITY;
        b200m_ebu_result z; memset (&z, 0, sizeof (z));
        z.loudness_M = z.maxloudn_M = z.loudness_S = z.maxloudn_S = z.integrated = z.integ_thr = z.range_min = z.range_max = z.range_thr = -200.0f;
        res[slot] = z;
    }
};

// bank control for this instance (all of a private bank, one slot of a shared one)
void bank_control (EbuPlugin* p, int cmd)
{
    if (!p->hub) { b200m_r128_control (p->bank, -1, cmd, nullptr); return; }
    std::lock_guard<std::mutex> lh (p->hub->mu);
    b200m_r128_control (p->hub->bank, p->slot, cmd, nullptr);
}

void send_control (EbuPlugin* p, int key, float value)       // forge_kvcontrolmessage, src/uris.h:279-294
{
    p->out.begin_event_object (p->u.control);
    p->out.prop_int (p->u.cckey, key);
    p->out.prop_float (p->u.ccval, value);
    p->out.end_object ();
}

void send_radarpoint (EbuPlugin* p, float m, float s, int pos)
{
    p->out.begin_event_object (p->u.rdr_radarpoint);
    p->out.prop_float (p->u.loudnessM, m);
    p->out.prop_float (p->u.loudnessS, s);
    p->out.prop_int (p->u.rdr_pointpos, pos);
    p->out.prop_int (p->u.rdr_pos_cur, p->radar_pos_cur);
    p->out.prop_int (p->u.rdr_pos_max, p->radar_pos_max);
    p->out.end_object ();
}

void set_radarspeed (EbuPlugin* p, float seconds)            // ebu_set_radarspeed (:75-78)
{
    p->radar_spd_max = (uint32_t)rint (seconds * p->rate / p->radar_pos_max);
    if (p->radar_spd_max < 4096) p->radar_spd_max = 4096;
}

float radartime (const EbuPlugin* p) { return (float)((uint32_t)p->radar_pos_max * p->radar_spd_max / p->rate); }

void forget_sent_histogram (EbuPlugin* p)
{
    for (int i = 0; i < HIST_LEN; ++i) { p->sentM[i] = 0; p->sentS[i] = 0; }
    p->hist_maxM = 0; p->hist_maxS = 0;
}

void reset_all (EbuPlugin* p)                                // ebu_reset (:45-61)
{
    bank_control (p, B200M_R128_RESET);
    send_control (p, CTL_LV2_RESETRADAR, 0);
    for (int i = 0; i < p->radar_pos_max; ++i) { p->radarS[i] = -INFINITY; p->radarM[i] = -INFINITY; }
    forget_sent_histogram (p);
    p->radar_pos_cur = 0;
    p->integration_time = 0;
}

void integrate (EbuPlugin* p, bool on)                       // ebu_integrate (:63-73)
{
    if (p->integrating == on) return;
    if (on) {
        if (p->follow_transport_mode & 2) reset_all (p);
        bank_control (p, B200M_R128_START);
    } else bank_control (p, B200M_R128_PAUSE);
    p->integrating = on;
}

void on_position (EbuPlugin* p, const AtomObject& obj)       // update_position (:84-113)
{
    const AtomHead* speed = obj.get (p->u.time_speed);
    if (!speed || speed->type != p->u.atom_Float || speed->size < 4) return;
    const float ts = *(const float*)(speed + 1);
    if (ts != 0 && !p->transport_rolling && (p->follow_transport_mode & 1)) integrate (p, true);
    if (ts == 0 && p->transport_rolling && (p->follow_transport_mode & 1)) integrate (p, false);
    p->transport_rolling = ts != 0;
}

void on_config (EbuPlugin* p, const AtomObject& obj, uint32_t n_samples)      // the metercfg switch (:283-327)
{
    const AtomHead* key = obj.get (p->u.cckey);
    const AtomHead* val = obj.get (p->u.ccval);
    if (!key || !val || key->size < 4 || val->size < 4) return;   // malformed message: key 0, ignored (src/uris.h:309-313)
    const int k = *(const int32_t*)(key + 1);
    const float v = *(const float*)(val + 1);
    switch (k) {
    case CTL_START: integrate (p, true); break;
    case CTL_PAUSE: integrate (p, false); break;
    case CTL_RESET: reset_all (p); break;
    case CTL_TRANSPORTSYNC:
        if (v == 1) { p->follow_transport_mode |= 1; if (p->transport_rolling != p->integrating) integrate (p, p->transport_rolling); }
        else p->follow_transport_mode &= ~1;
        break;
    case CTL_AUTORESET:
        if (v == 1) p->follow_transport_mode |= 2; else p->follow_transport_mode &= ~2;
        break;
    case CTL_RADARTIME:
        if (v >= 30 && v <= 600) { set_radarspeed (p, v); if (p->radar_spd_max < 2 * n_samples) p->radar_spd_max = 2 * n_samples; }
        send_control (p, CTL_LV2_RADARTIME, radartime (p));
        break;
    case CTL_UISETTINGS:
        p->ui_settings = (uint32_t)v;
        p->dbtp_enable = (p->ui_settings & 64) != 0;
        break;
    default: break;
    }
}

LV2_Handle ebur_instantiate (const LV2_Descriptor* d, double rate, const char*, const LV2_Feature* const* features)
{
    if (strcmp (d->URI, MTR_URI "EBUr128")) return nullptr;
    const LV2_URID_Map* map = find_urid_map (features);
    if (!map) { fprintf (stderr, "EBUrLV2 error: Host does not support urid:map\n"); return nullptr; }      // :140-144
    EbuPlugin* p = new (std::nothrow) EbuPlugin;
    if (!p) return nullptr;
    auto M = [&] (const char* uri) { return map->map (map->handle, uri); };
    Urids& u = p->u;
    u.atom_Blank = M (B200M_LV2_ATOM "Blank"); u.atom_Object = M (B200M_LV2_ATOM "Object"); u.atom_Int = M (B200M_LV2_ATOM "Int");
    u.atom_Float = M (B200M_LV2_ATOM "Float"); u.atom_Bool = M (B200M_LV2_ATOM "Bool"); u.atom_Sequence = M (B200M_LV2_ATOM "Sequence");
    u.time_Position = M (B200M_LV2_TIME "Position"); u.time_speed = M (B200M_LV2_TIME "speed");
    u.ebulevels = M (MTR_URI "ebulevels"); u.loudnessM = M (MTR_URI "ebu_loudnessM"); u.maxloudnM = M (MTR_URI "ebu_maxloudnM");
    u.loudnessS = M (MTR_URI "ebu_loudnessS"); u.maxloudnS = M (MTR_URI "ebu_maxloudnS"); u.integrated = M (MTR_URI "ebu_integrated");
    u.range_min = M (MTR_URI "ebu_range_min"); u.range_max = M (MTR_URI "ebu_range_max"); u.integrating = M (MTR_URI "ebu_integrating");
    u.integr_time = M (MTR_URI "ebu_integr_time"); u.ebu_state = M (MTR_URI "ebu_state");
    u.rdr_histogram = M (MTR_URI "rdr_histogram"); u.rdr_histpoint = M (MTR_URI "rdr_histpoint"); u.rdr_radarpoint = M (MTR_URI "rdr_radarpoint");
    u.rdr_pointpos = M (MTR_URI "rdr_pointpos"); u.rdr_pos_cur = M (MTR_URI "rdr_pos_cur"); u.rdr_pos_max = M (MTR_URI "rdr_pos_max");
    u.truepeak = M (MTR_URI "truepeak");
    u.cckey = M (MTR_URI "controlkey"); u.ccval = M (MTR_URI "controlval"); u.control = M (MTR_URI "control");
    u.meteron = M (MTR_URI "meteron"); u.meteroff = M (MTR_URI "meteroff"); u.metercfg = M (MTR_URI "metercfg");
    p->out.t_sequence = u.atom_Sequence; p->out.t_object = u.atom_Object; p->out.t_int = u.atom_Int; p->out.t_float = u.atom_Float; p->out.t_bool = u.atom_Bool;
    p->rate = rate;
    for (int i = 0; i < RADAR_POINTS; ++i) { p->radarS[i] = -INFINITY; p->radarM[i] = -INFINITY; }
    set_radarspeed (p, 2.0 * 60.0);
    forget_sent_histogram (p);
    p->hub = (EbuHub*)SlotHub::join (HubKey{HUB_EBUR128, 0, 2, 0, rate}, p, &p->slot, EbuHub::create);
    if (!p->hub) {
        if (b200m_r128_create (&p->bank, 0, 1, (float)rate, 0)) { delete p; return nullptr; }     // ebu->init (2, rate); 2 x TruePeakdsp (:189-196)
        p->stage.reserve (2);
    }
    return p;
}

void ebur_connect (LV2_Handle h, uint32_t port, void* data)
{
    EbuPlugin* p = (EbuPlugin*)h;
    switch (port) {
    case EBU_CONTROL: p->control = data; break;
    case EBU_NOTIFY:  p->notify = data; break;
    case EBU_INPUT0:  p->input[0] = (float*)data; break;
    case EBU_OUTPUT0: p->output[0] = (float*)data; break;
    case EBU_INPUT1:  p->input[1] = (float*)data; break;
    case EBU_OUTPUT1: p->output[1] = (float*)data; break;
    default: break;
    }
}

bool fetch_histogram (EbuPlugin* p)
{
    if (!p->hub) return b200m_r128_histogram (p->bank, 0, p->histM, p->histS, nullptr) == 0;
    std::lock_guard<std::mutex> lh (p->hub->mu);               // waits for a cycle in flight: only instances with an open UI pay this
    return b200m_r128_histogram (p->hub->bank, (uint32_t)p->slot, p->histM, p->histS, nullptr) == 0;
}

void ebur_run (LV2_Handle h, uint32_t n_samples)
{
    EbuPlugin* p = (EbuPlugin*)h;
    // audio first, whatever happens to the metering below (the reference ends ebur128_run with this copy, src/ebulv2.cc:484-491;
    // doing it first means an engine failure, a missing notify port or an over-long cycle can never drop audio)
    forward_audio (p->input, p->output, 2, n_samples);
    if (!p->notify || !p->input[0] || !p->input[1]) return;
    const uint32_t capacity = ((const AtomHead*)p->notify)->size;      // host convention: capacity of the output port
    p->out.begin_sequence (p->notify, capacity);

    if (p->send_state_to_ui && p->ui_active) {
        p->send_state_to_ui = false;
        send_control (p, CTL_LV2_FTM, (float)p->follow_transport_mode);
        send_control (p, CTL_LV2_RADARTIME, radartime (p));
        send_control (p, CTL_UISETTINGS, (float)p->ui_settings);
    }

    if (p->hub && n_samples >= 1 && n_samples <= B200M_MAX_BLOCK) {
        // close a cycle this run() breaks BEFORE this cycle's control messages reach the bank, so that a RESET / START meant for
        // the new cycle does not land ahead of the old audio
        std::lock_guard<std::mutex> lh (p->hub->mu);
        p->hub->close_if_broken (p->slot, n_samples);
        p->hub->first_run (p->slot);
    }
    if (p->control) {                                          // messages from the GUI / host (:258-331)
        for (AtomEvents ev (p->control); ev.valid (); ev.next ()) {
            const AtomHead* a = ev.body ();
            if (a->type != p->u.atom_Blank && a->type != p->u.atom_Object) continue;
            AtomObject obj; obj.a = a;
            const uint32_t ot = obj.otype ();
            if (ot == p->u.time_Position) on_position (p, obj);
            else if (ot == p->u.meteron) { p->ui_active = true; p->send_state_to_ui = true; p->radar_resync = 0; forget_sent_histogram (p); }
            else if (ot == p->u.meteroff) p->ui_active = false;
            else if (ot == p->u.metercfg) on_config (p, obj, n_samples);
        }
    }

    // ---- audio cycle on the GPU (:341-367) ----------------------------------------------------------------------
    b200m_ebu_result r; float tp_max = -INFINITY;
    memset (&r, 0, sizeof (r));
    bool ran = false;
    if (p->hub && n_samples >= 1 && n_samples <= B200M_MAX_BLOCK) {
        EbuHub* hub = p->hub;
        std::lock_guard<std::mutex> lh (hub->mu);
        hub->submit (p->slot, p->input, n_samples);
        r = hub->res[p->slot]; tp_max = hub->tp[p->slot];      // the previous cycle's (-inf if the slot's dBTP was off in it)
        ran = true;
    } else if (n_samples >= 1 && n_samples <= B200M_MAX_BLOCK && p->stage.fill (p->input, 2, n_samples)) {
        b200m_r128_set_dbtp (p->bank, p->dbtp_enable);
        ran = b200m_r128_run_host (p->bank, p->stage.data, p->stage.cap, n_samples) == 0 && b200m_r128_results (p->bank, &r, &tp_max, nullptr) == 0;
    }
    if (!ran) return;                                          // run() never fails: leave the (empty) sequence
    const float lm = r.loudness_M, mm = r.maxloudn_M, ls = r.loudness_S, ms = r.maxloudn_S, il = r.integrated, rn = r.range_min, rx = r.range_max;

    if (p->radar_resync >= 0) {                                // replay the stored radar to a GUI that just connected (:369-389)
        int batch = (int)((capacity - 512u) / 192u);             // unsigned, as in the reference's expression
        if (batch > 16) batch = 16;
        for (int i = 0; i < batch; ++i, ++p->radar_resync) {
            if (p->radar_resync >= p->radar_pos_max) { p->radar_resync = -1; send_control (p, CTL_LV2_RESYNCDONE, 0); break; }
            send_radarpoint (p, p->radarM[p->radar_resync], p->radarS[p->radar_resync], p->radar_resync);
        }
    }

    if (lm > p->radarMC) p->radarMC = lm;                      // radar history (:391-393; the second test reads lm, as there)
    if (lm > p->radarSC) p->radarSC = ls;
    if (p->integrating) p->integration_time += n_samples;
    p->radar_spd_cur += n_samples;
    if (p->radar_spd_cur > p->radar_spd_max) {
        if (p->ui_active) send_radarpoint (p, p->radarMC, p->radarSC, p->radar_pos_cur);
        p->radarM[p->radar_pos_cur] = p->radarMC;
        p->radarS[p->radar_pos_cur] = p->radarSC;
        p->radar_spd_cur = p->radar_spd_cur % p->radar_spd_max;
        p->radar_pos_cur = (p->radar_pos_cur + 1) % p->radar_pos_max;
        p->radarSC = p->radarMC = -INFINITY;
    }

    if (p->ui_active && r.hist_M_count > 10 && r.hist_S_count > 10 &&
        fetch_histogram (p)) {                                                                // histogram deltas (:420-461)
        int msgtx = 0; bool max_changed = false;
        for (int i = 110; i < 650; ++i) {
            const int vm = p->histM[i], vs = p->histS[i];
            if (capacity - p->out.sequence_size () <= 512) break;
            if (p->sentM[i] != vm || p->sentS[i] != vs) {
                if (msgtx++ > 16) break;
                p->sentM[i] = vm; p->sentS[i] = vs;
                p->out.begin_event_object (p->u.rdr_histpoint);
                p->out.prop_int (p->u.loudnessM, vm);
                p->out.prop_int (p->u.loudnessS, vs);
                p->out.prop_int (p->u.rdr_pointpos, i);
                p->out.end_object ();
            }
            if (vm > p->hist_maxM) { p->hist_maxM = vm; max_changed = true; }
            if (vs > p->hist_maxS) { p->hist_maxS = vs; max_changed = true; }
        }
        if (max_changed) {
            p->out.begin_event_object (p->u.rdr_histogram);
            p->out.prop_int (p->u.loudnessM, p->hist_maxM);
            p->out.prop_int (p->u.loudnessS, p->hist_maxS);
            p->out.end_object ();
        }
    }

    if (p->ui_active) {                                        // ebulevels (:464-482)
        p->out.begin_event_object (p->u.ebulevels);
        p->out.prop_float (p->u.loudnessM, lm);
        p->out.prop_float (p->u.maxloudnM, mm);
        p->out.prop_float (p->u.loudnessS, ls);
        p->out.prop_float (p->u.maxloudnS, ms);
        p->out.prop_float (p->u.integrated, il);
        p->out.prop_float (p->u.range_min, rn);
        p->out.prop_float (p->u.range_max, rx);
        p->out.prop_float (p->u.truepeak, tp_max);
        p->out.prop_bool (p->u.integrating, p->integrating);
        p->out.prop_float (p->u.integr_time, (float)(p->integration_time / p->rate));
        p->out.end_object ();
    }
}

void ebur_cleanup (LV2_Handle h)
{
    EbuPlugin* p = (EbuPlugin*)h;
    if (p->hub) p->hub->leave (p->slot); else b200m_r128_destroy (p->bank);
    p->stage.release ();
    delete p;
}

// LV2 state extension (:513-548): flags = LV2_STATE_IS_POD | LV2_STATE_IS_PORTABLE, status 0 = LV2_STATE_SUCCESS
uint32_t ebur_save (LV2_Handle h, LV2_State_Store_Function store, void* handle, uint32_t, const LV2_Feature* const*)
{
    EbuPlugin* p = (EbuPlugin*)h;
    uint32_t cfg = p->ui_settings;
    cfg |= (uint32_t)p->follow_transport_mode << 8;
    cfg |= p->radar_spd_max << 16;
    store (handle, p->u.ebu_state, &cfg, sizeof (uint32_t), p->u.atom_Int, 1u | 2u);
    return 0;
}

uint32_t ebur_restore (LV2_Handle h, LV2_State_Retrieve_Function retrieve, void* handle, uint32_t, const LV2_Feature* const*)
{
    EbuPlugin* p = (EbuPlugin*)h;
    size_t size = 0; uint32_t type = 0, vflags = 0;
    const void* value = retrieve (handle, p->u.ebu_state, &size, &type, &vflags);
    if (value && size == sizeof (uint32_t) && type == p->u.atom_Int) {
        const uint32_t cfg = *(const uint32_t*)value;
        p->ui_settings = cfg & 0xff;
        p->follow_transport_mode = (cfg >> 8) & 0x3;
        p->radar_spd_max = cfg >> 16;
        p->dbtp_enable = (p->ui_settings & 64) != 0;
        p->send_state_to_ui = true;
    }
    return 0;
}

const void* ebur_extension_data (const char* uri)
{
    static const LV2_State_Interface state = {ebur_save, ebur_restore};
    return strcmp (uri, B200M_LV2_STATE_INTERFACE) ? nullptr : &state;
}

const LV2_Descriptor g_ebur128 = {MTR_URI "EBUr128", ebur_instantiate, ebur_connect, nullptr, ebur_run, nullptr, ebur_cleanup, ebur_extension_data};

}  // namespace

namespace b200m { const LV2_Descriptor* lv2_ebur128_descriptor () { return &g_ebur128; } }
