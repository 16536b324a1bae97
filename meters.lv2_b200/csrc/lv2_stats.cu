// lv2_stats.cu — the "bitmeter" and "SigDistHist" plugins (descriptors 31 and 29 of the reference, src/meters.cc:779,777)
// over one-instance b200m_bim / b200m_sdh banks, or one slot of a shared bank in batched mode (StatsHub): same URIs, ports,
// control messages, notify-port messages and state extension as src/bitmeter.c:108-388 and src/sigdistlv2.c:108-445.
// The per-sample scans and the bit-meter's ~5 fps window run on the GPU; the 25 fps SigDistHist cadence, the transport-follow
// logic and the message forging are host code restated from those files, message for message (tests/test_lv2_stats_gpu.py
// compares the notify buffers byte for byte).
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "lv2_hub.cuh"

namespace {

using namespace b200m;

// numeric control keys, src/uris.h:187-203
enum { CTL_START = 1, CTL_PAUSE, CTL_RESET, CTL_TRANSPORTSYNC, CTL_AUTORESET, CTL_RADARTIME, CTL_UISETTINGS,
       CTL_LV2_RADARTIME, CTL_LV2_FTM, CTL_LV2_RESETRADAR, CTL_LV2_RESYNCDONE, CTL_SAMPLERATE, CTL_WINDOWED, CTL_AVERAGE };
constexpr int BIM_LAST = 584, DIST_BIN = 361;                  // src/uris.h:49,60

// the statistics of n bit-meter instances as one b200m_bim_results_all call leaves them (row layouts: include/b200meters.h)
struct BimRows {
    std::vector<int32_t> hist, cnt, closed, pub_hist, pub_cnt; std::vector<float> mm, pub_mm; std::vector<int64_t> itime, pub_itime;
    void resize (uint32_t n)
    {
        hist.resize ((size_t)n * BIM_LAST); cnt.resize (n * 5); mm.resize (n * 2); itime.resize (n); closed.resize (n);
        pub_hist.resize ((size_t)n * BIM_LAST); pub_cnt.resize (n * 5); pub_mm.resize (n * 2); pub_itime.resize (n);
    }
    // live / pub: which statistics to read (with both, the closed flags too); one synchronisation whatever is read
    int collect (b200m_bim* b, bool live, bool pub)
    {
        return b200m_bim_results_all (b, live ? hist.data () : nullptr, live ? cnt.data () : nullptr, live ? mm.data () : nullptr, live ? itime.data () : nullptr,
                                      live && pub ? closed.data () : nullptr, pub ? pub_hist.data () : nullptr, pub ? pub_cnt.data () : nullptr,
                                      pub ? pub_mm.data () : nullptr, pub ? pub_itime.data () : nullptr, nullptr);
    }
};
struct SdhRows {
    std::vector<int32_t> hist, mp; std::vector<double> av; std::vector<int64_t> itime;
    void resize (uint32_t n) { hist.resize ((size_t)n * DIST_BIN); mp.resize (n * 2); av.resize (n * 3); itime.resize (n); }
    int collect (b200m_sdh* b, bool live)
    {
        return b200m_sdh_results_all (b, live ? hist.data () : nullptr, live ? mp.data () : nullptr, live ? av.data () : nullptr, live ? itime.data () : nullptr, nullptr);
    }
};

// batched mode (lv2_hub.cuh): the bitmeter instances of one sample rate share one b200m_bim bank, the SigDistHist instances one
// b200m_sdh bank.  Every slot has its own control state on the device, so START / PAUSE / RESET / AVERAGE / WINDOWED and the
// bit-meter's window clock stay per instance.
struct StatsHub : SlotHub {
    b200m_bim* bim = nullptr; b200m_sdh* sdh = nullptr;
    BimRows br; SdhRows sr;                                    // the last completed cycle

    StatsHub (const HubKey& k, uint32_t n) : SlotHub (k, n) {}
    ~StatsHub () { b200m_bim_destroy (bim); b200m_sdh_destroy (sdh); }

    static SlotHub* create (const HubKey& k, uint32_t n)
    {
        StatsHub* h = new (std::nothrow) StatsHub (k, n);
        if (!h) return nullptr;
        const bool is_bim = k.family == HUB_BITMETER;
        if (is_bim ? b200m_bim_create (&h->bim, 0, n, k.rate) : b200m_sdh_create (&h->sdh, 0, n, k.rate)) { delete h; return nullptr; }
        if (is_bim) h->br.resize (n); else h->sr.resize (n);
        return h;
    }
    int launch_bank (uint32_t n) override
    {
        return bim ? b200m_bim_run_host (bim, stage.data, B200M_MAX_BLOCK, n) : b200m_sdh_run_host (sdh, stage.data, B200M_MAX_BLOCK, n);
    }
    void collect () override { if (bim) br.collect (bim, true, true); else sr.collect (sdh, true); }
    // the slot's next tenant starts from a freshly instantiated plugin (bit-meter: bim_reset, integrating, windowed, window clock
    // at 0; SigDistHist: sdh_reset, integration off)
    void vacate (uint32_t slot) override { control ((int32_t)slot, B200M_CTL_CLEAR); }
    int control (int32_t slot, int cmd) { return bim ? b200m_bim_control_inst (bim, slot, cmd, nullptr) : b200m_sdh_control_inst (sdh, slot, cmd, nullptr); }
};

// run() decides in cycle k whether cycle k's statistics are published, from the flags as they stood then; a private instance
// forges the events in the same run(), a batched one in cycle k + 1, when cycle k's statistics have been collected
struct Cycle {
    bool valid = false, ui_active = false, integrating = false, averaging = false, send_state = false;
    bool due = false;                                          // SigDistHist: the 25 fps cadence fired and a UI listens
};

struct StatsPlugin {
    bool is_bim = false;
    b200m_bim* bim = nullptr; b200m_sdh* sdh = nullptr;       // private bank of one, or slot `slot` of hub's bank
    StatsHub* hub = nullptr; int slot = -1;
    PinnedStage stage; BimRows br; SdhRows sr;                // private bank only
    Cycle last;                                                // batched: the previous cycle's decision
    bool mode_dirty = false;                                   // bitmeter: a restored AVERAGE / WINDOWED reaches the bank with the next run()
    AtomWriter out;
    const void* control = nullptr; void* notify = nullptr;
    float* input[2] = {nullptr, nullptr}; float* output[2] = {nullptr, nullptr};
    double rate = 48000;
    bool ui_active = false, send_state_to_ui = false, integrating = false, averaging = false, transport_rolling = false;
    int follow_transport_mode = 0, radar_resync = 0;
    uint32_t ui_settings = 0;
    struct {
        LV2_URID atom_Blank, atom_Object, atom_Int, atom_Float, time_Position, time_speed;
        LV2_URID control, cckey, ccval, meteron, meteroff, metercfg, integrating, integr_time, sdh_state, bim_state;
        LV2_URID sdh_histogram, sdh_hist_max, sdh_hist_var, sdh_hist_avg, sdh_hist_peak, sdh_hist_data, sdh_information;
        LV2_URID bim_information, bim_averaging, bim_stats, bim_data, bim_zero, bim_pos, bim_min, bim_max, bim_nan, bim_inf, bim_den;
    } u;
};

// bank control for this instance (all of a private bank, one slot of a shared one)
void bank_control (StatsPlugin* p, int cmd)
{
    if (!p->hub) { if (p->is_bim) b200m_bim_control (p->bim, cmd, nullptr); else b200m_sdh_control (p->sdh, cmd, nullptr); return; }
    std::lock_guard<std::mutex> lh (p->hub->mu);
    p->hub->control (p->slot, cmd);
}

Cycle this_cycle (const StatsPlugin* p, bool due)
{
    Cycle c;
    c.valid = true; c.ui_active = p->ui_active; c.integrating = p->integrating; c.averaging = p->averaging; c.send_state = p->send_state_to_ui; c.due = due;
    return c;
}

void send_control (StatsPlugin* p, int key, float value)       // forge_kvcontrolmessage, src/uris.h:279-294
{
    p->out.begin_event_object (p->u.control);
    p->out.prop_int (p->u.cckey, key);
    p->out.prop_float (p->u.ccval, value);
    p->out.end_object ();
}

bool read_cfg (StatsPlugin* p, const AtomObject& obj, int* k, float* v)
{
    const AtomHead* key = obj.get (p->u.cckey);
    const AtomHead* val = obj.get (p->u.ccval);
    if (!key || !val || key->size < 4 || val->size < 4) return false;   // malformed: key 0, ignored (src/uris.h:309-313)
    *k = *(const int32_t*)(key + 1); *v = *(const float*)(val + 1);
    return true;
}

// ---- SigDistHist helpers (src/sigdistlv2.c:50-105) ----------------------------------------------------------------
void sdh_reset (StatsPlugin* p)
{
    send_control (p, CTL_LV2_RESETRADAR, 0);
    bank_control (p, B200M_CTL_RESET);
    p->radar_resync = 0;
}

void sdh_integrate (StatsPlugin* p, bool on)
{
    if (p->integrating == on) return;
    if (on && (p->follow_transport_mode & 2)) sdh_reset (p);
    bank_control (p, on ? B200M_CTL_START : B200M_CTL_PAUSE);
    p->integrating = on;
}

void sdh_position (StatsPlugin* p, const AtomObject& obj)
{
    const AtomHead* speed = obj.get (p->u.time_speed);
    if (!speed || speed->type != p->u.atom_Float || speed->size < 4) return;
    const float ts = *(const float*)(speed + 1);
    if (ts != 0 && !p->transport_rolling && (p->follow_transport_mode & 1)) sdh_integrate (p, true);
    if (ts == 0 && p->transport_rolling && (p->follow_transport_mode & 1)) sdh_integrate (p, false);
    p->transport_rolling = ts != 0;
}

LV2_Handle stats_instantiate (const LV2_Descriptor* d, double rate, const char*, const LV2_Feature* const* features)
{
    const bool is_bim = !strcmp (d->URI, MTR_URI "bitmeter");
    if (!is_bim && strcmp (d->URI, MTR_URI "SigDistHist")) return nullptr;
    const LV2_URID_Map* map = find_urid_map (features);
    if (!map) { fprintf (stderr, "%s error: Host does not support urid:map\n", is_bim ? "Bitmeter" : "SigDistHist"); return nullptr; }
    StatsPlugin* p = new (std::nothrow) StatsPlugin;
    if (!p) return nullptr;
    p->is_bim = is_bim; p->rate = rate;
    auto M = [&] (const char* uri) { return map->map (map->handle, uri); };
    auto& u = p->u;
    u.atom_Blank = M (B200M_LV2_ATOM "Blank"); u.atom_Object = M (B200M_LV2_ATOM "Object"); u.atom_Int = M (B200M_LV2_ATOM "Int"); u.atom_Float = M (B200M_LV2_ATOM "Float");
    u.time_Position = M (B200M_LV2_TIME "Position"); u.time_speed = M (B200M_LV2_TIME "speed");
    u.control = M (MTR_URI "control"); u.cckey = M (MTR_URI "controlkey"); u.ccval = M (MTR_URI "controlval");
    u.meteron = M (MTR_URI "meteron"); u.meteroff = M (MTR_URI "meteroff"); u.metercfg = M (MTR_URI "metercfg");
    u.integrating = M (MTR_URI "ebu_integrating"); u.integr_time = M (MTR_URI "ebu_integr_time");
    u.sdh_state = M (MTR_URI "sdh_state"); u.bim_state = M (MTR_URI "bim_state");
    u.sdh_histogram = M (MTR_URI "sdh_histogram"); u.sdh_hist_max = M (MTR_URI "sdh_hist_max"); u.sdh_hist_var = M (MTR_URI "sdh_hist_var");
    u.sdh_hist_avg = M (MTR_URI "sdh_hist_avg"); u.sdh_hist_peak = M (MTR_URI "sdh_hist_peak"); u.sdh_hist_data = M (MTR_URI "sdh_hist_data");
    u.sdh_information = M (MTR_URI "sdh_information");
    u.bim_information = M (MTR_URI "bim_information"); u.bim_averaging = M (MTR_URI "bim_averaging"); u.bim_stats = M (MTR_URI "bim_stats");
    u.bim_data = M (MTR_URI "bim_data"); u.bim_zero = M (MTR_URI "bim_zero"); u.bim_pos = M (MTR_URI "bim_pos"); u.bim_min = M (MTR_URI "bim_min");
    u.bim_max = M (MTR_URI "bim_max"); u.bim_nan = M (MTR_URI "bim_nan"); u.bim_inf = M (MTR_URI "bim_inf"); u.bim_den = M (MTR_URI "bim_den");
    p->out.t_sequence = M (B200M_LV2_ATOM "Sequence"); p->out.t_object = u.atom_Object; p->out.t_int = u.atom_Int; p->out.t_float = u.atom_Float;
    p->out.t_bool = M (B200M_LV2_ATOM "Bool"); p->out.t_long = M (B200M_LV2_ATOM "Long"); p->out.t_double = M (B200M_LV2_ATOM "Double");
    p->out.t_vector = M (B200M_LV2_ATOM "Vector");
    p->integrating = is_bim;                                   // src/bitmeter.c:150-151, src/sigdistlv2.c:141-150
    p->hub = (StatsHub*)SlotHub::join (HubKey{is_bim ? HUB_BITMETER : HUB_SIGDIST, 0, 1, 0, rate}, p, &p->slot, StatsHub::create);
    if (p->hub) {
        // a fresh instance whatever the slot metered while it was vacant: the bit-meter's window clock starts at 0 with this run()
        bank_control (p, B200M_CTL_CLEAR);
        return p;
    }
    const int rc = is_bim ? b200m_bim_create (&p->bim, 0, 1, rate) : b200m_sdh_create (&p->sdh, 0, 1, rate);
    if (rc) { delete p; return nullptr; }
    p->stage.reserve (1);
    if (is_bim) p->br.resize (1); else p->sr.resize (1);
    return p;
}

void stats_connect (LV2_Handle h, uint32_t port, void* data)
{
    StatsPlugin* p = (StatsPlugin*)h;
    switch (port) {                                            // BIMPortIndex / SDHPortIndex
    case 0: p->control = data; break;
    case 1: p->notify = data; break;
    case 2: p->input[0] = (float*)data; break;
    case 3: p->output[0] = (float*)data; break;
    case 4: p->input[1] = (float*)data; break;                // SigDistHist declares a second, unused audio pair
    case 5: p->output[1] = (float*)data; break;
    default: break;
    }
}

bool stage_block (StatsPlugin* p, uint32_t n)
{
    return n >= 1 && n <= B200M_MAX_BLOCK && p->stage.fill (p->input, 1, n);
}

bool valid_block (uint32_t n) { return n >= 1 && n <= B200M_MAX_BLOCK; }

// with a hub: close a cycle this run() breaks BEFORE this cycle's control messages reach the bank (as ebur_run does), so that a
// RESET / START meant for the new cycle does not land ahead of the old audio
void close_if_broken (StatsPlugin* p, uint32_t n)
{
    if (!p->hub || !valid_block (n)) return;
    std::lock_guard<std::mutex> lh (p->hub->mu);
    p->hub->close_if_broken (p->slot, n);
}

// bim_stats / bim_information of one cycle (src/bitmeter.c:267-327): `closed` = that cycle closed the instance's window
void bim_publish (StatsPlugin* p, const Cycle& c, bool closed, const BimRows& r, uint32_t i)
{
    if (!(closed || c.send_state)) return;
    if (c.ui_active && (c.integrating || c.send_state)) {
        const int32_t* cnt = (closed ? r.pub_cnt.data () : r.cnt.data ()) + 5 * i;
        const float* mm = (closed ? r.pub_mm.data () : r.mm.data ()) + 2 * i;
        p->out.begin_event_object (p->u.bim_stats);
        p->out.prop_long (p->u.integr_time, closed ? r.pub_itime[i] : r.itime[i]);
        p->out.prop_int (p->u.bim_zero, cnt[0]);
        p->out.prop_int (p->u.bim_pos, cnt[1]);
        p->out.prop_double (p->u.bim_max, mm[1]);
        p->out.prop_double (p->u.bim_min, mm[0]);
        p->out.prop_int (p->u.bim_nan, cnt[2]);
        p->out.prop_int (p->u.bim_inf, cnt[3]);
        p->out.prop_int (p->u.bim_den, cnt[4]);
        p->out.prop_vector_i32 (p->u.bim_data, (closed ? r.pub_hist.data () : r.hist.data ()) + (size_t)i * BIM_LAST, BIM_LAST);
        p->out.end_object ();
    }
    if (closed && c.ui_active) {
        p->out.begin_event_object (p->u.bim_information);
        p->out.prop_bool (p->u.integrating, c.integrating);
        p->out.prop_bool (p->u.bim_averaging, c.averaging);
        p->out.end_object ();
    }
}

void bim_run (StatsPlugin* p, uint32_t n)
{
    if (p->send_state_to_ui && p->ui_active) { p->send_state_to_ui = false; send_control (p, CTL_SAMPLERATE, (float)p->rate); }
    close_if_broken (p, n);
    if (p->mode_dirty) { p->mode_dirty = false; bank_control (p, p->averaging ? B200M_CTL_AVERAGE : B200M_CTL_WINDOWED); }
    if (p->control) {                                          // src/bitmeter.c:197-236
        for (AtomEvents ev (p->control); ev.valid (); ev.next ()) {
            const AtomHead* a = ev.body ();
            if (a->type != p->u.atom_Blank && a->type != p->u.atom_Object) continue;
            AtomObject obj; obj.a = a;
            const uint32_t ot = obj.otype ();
            if (ot == p->u.meteron) { p->ui_active = true; p->send_state_to_ui = true; }
            else if (ot == p->u.meteroff) p->ui_active = false;
            else if (ot == p->u.metercfg) {
                int k = 0; float v = 0;
                if (!read_cfg (p, obj, &k, &v)) continue;
                switch (k) {
                case CTL_START: p->integrating = true; bank_control (p, B200M_CTL_START); break;
                case CTL_PAUSE: p->integrating = false; bank_control (p, B200M_CTL_PAUSE); break;
                case CTL_RESET: bank_control (p, B200M_CTL_RESET); p->send_state_to_ui = true; break;
                case CTL_AVERAGE: p->averaging = true; bank_control (p, B200M_CTL_AVERAGE); break;
                case CTL_WINDOWED: p->averaging = false; bank_control (p, B200M_CTL_WINDOWED); break;
                default: break;
                }
            }
        }
    }
    const Cycle now = this_cycle (p, false);
    if (p->hub) {
        if (!valid_block (n)) { p->last.valid = false; return; }
        std::lock_guard<std::mutex> lh (p->hub->mu);
        p->hub->submit (p->slot, p->input, n);
        if (p->last.valid) bim_publish (p, p->last, p->hub->br.closed[p->slot] != 0, p->hub->br, (uint32_t)p->slot);      // the previous cycle's
        p->last = now;
        return;
    }
    if (!stage_block (p, n) || b200m_bim_run_host (p->bim, p->stage.data, p->stage.cap, n)) return;
    // run() is synchronous for the host: the staging block is rewritten next cycle, so the asynchronous upload and the scan
    // must have finished before we return even when nothing is published (a collect that reads nothing = stream sync)
    const bool closed = b200m_bim_window_closed (p->bim) != 0;
    const bool stats = (closed || now.send_state) && now.ui_active && (now.integrating || now.send_state);
    if (p->br.collect (p->bim, stats && !closed, stats && closed)) return;
    bim_publish (p, now, closed, p->br, 0);
}

// sdh_histogram / sdh_information of one cycle (src/sigdistlv2.c:329-350), when that cycle's 25 fps cadence fired for a UI
void sdh_publish (StatsPlugin* p, const Cycle& c, const SdhRows& r, uint32_t i)
{
    if (!c.due) return;
    if (c.integrating || c.send_state) {
        p->out.begin_event_object (p->u.sdh_histogram);
        p->out.prop_int (p->u.sdh_hist_max, r.mp[2 * i]);
        p->out.prop_double (p->u.sdh_hist_avg, r.av[3 * i]);
        p->out.prop_double (p->u.sdh_hist_var, r.av[3 * i + 2]);
        p->out.prop_int (p->u.sdh_hist_peak, r.mp[2 * i + 1]);
        p->out.prop_vector_i32 (p->u.sdh_hist_data, r.hist.data () + (size_t)i * DIST_BIN, DIST_BIN);
        p->out.end_object ();
    }
    p->out.begin_event_object (p->u.sdh_information);
    p->out.prop_bool (p->u.integrating, c.integrating);
    p->out.prop_long (p->u.integr_time, r.itime[i]);
    p->out.end_object ();
}

// the 25 fps cadence of a cycle of n frames (:329-331): true when this cycle publishes to a listening UI
bool sdh_due (StatsPlugin* p, uint32_t n)
{
    const double lim = p->rate / 25.f;                         // const int fps_limit = MAX (rate / 25.f, n_samples)  (:329)
    const int fps_limit = (int)(lim > n ? lim : (double)n);
    p->radar_resync += (int)n;
    if (!(p->radar_resync >= fps_limit || p->send_state_to_ui)) return false;
    p->radar_resync = p->radar_resync % fps_limit;
    return p->ui_active;
}

void sdh_run (StatsPlugin* p, uint32_t n)
{
    if (p->send_state_to_ui && p->ui_active) {                 // src/sigdistlv2.c:205-210
        p->send_state_to_ui = false;
        send_control (p, CTL_LV2_FTM, (float)p->follow_transport_mode);
        send_control (p, CTL_SAMPLERATE, (float)p->rate);
        send_control (p, CTL_UISETTINGS, (float)p->ui_settings);
    }
    close_if_broken (p, n);
    if (p->control) {                                          // :213-271
        for (AtomEvents ev (p->control); ev.valid (); ev.next ()) {
            const AtomHead* a = ev.body ();
            if (a->type != p->u.atom_Blank && a->type != p->u.atom_Object) continue;
            AtomObject obj; obj.a = a;
            const uint32_t ot = obj.otype ();
            if (ot == p->u.time_Position) sdh_position (p, obj);
            else if (ot == p->u.meteron) { p->ui_active = true; p->send_state_to_ui = true; }
            else if (ot == p->u.meteroff) p->ui_active = false;
            else if (ot == p->u.metercfg) {
                int k = 0; float v = 0;
                if (!read_cfg (p, obj, &k, &v)) continue;
                switch (k) {
                case CTL_START: sdh_integrate (p, true); break;
                case CTL_PAUSE: sdh_integrate (p, false); break;
                case CTL_RESET: sdh_reset (p); break;
                case CTL_TRANSPORTSYNC:
                    if (v == 1) { p->follow_transport_mode |= 1; if (p->transport_rolling != p->integrating) sdh_integrate (p, p->transport_rolling); }
                    else p->follow_transport_mode &= ~1;
                    break;
                case CTL_AUTORESET: if (v == 1) p->follow_transport_mode |= 2; else p->follow_transport_mode &= ~2; break;
                case CTL_UISETTINGS: p->ui_settings = (uint32_t)v; break;
                default: break;
                }
            }
        }
    }
    if (p->hub) {
        if (!valid_block (n)) { p->last.valid = false; return; }
        std::lock_guard<std::mutex> lh (p->hub->mu);
        p->hub->submit (p->slot, p->input, n);
        if (p->last.valid) sdh_publish (p, p->last, p->hub->sr, (uint32_t)p->slot);                                       // the previous cycle's
        p->last = this_cycle (p, sdh_due (p, n));
        return;
    }
    if (!stage_block (p, n) || b200m_sdh_run_host (p->sdh, p->stage.data, p->stage.cap, n)) return;
    const Cycle now = this_cycle (p, sdh_due (p, n));
    if (p->sr.collect (p->sdh, now.due)) return;              // synchronous run(), see bim_run
    sdh_publish (p, now, p->sr, 0);
}

void stats_run (LV2_Handle h, uint32_t n)
{
    StatsPlugin* p = (StatsPlugin*)h;
    // audio first (src/bitmeter.c:330-334, src/sigdistlv2.c:372-376 end with this copy): a metering failure never drops it
    forward_audio (p->input, p->output, 1, n);
    if (!p->notify || !p->input[0]) return;
    p->out.begin_sequence (p->notify, ((const AtomHead*)p->notify)->size);
    if (p->is_bim) bim_run (p, n); else sdh_run (p, n);
}

void stats_cleanup (LV2_Handle h)
{
    StatsPlugin* p = (StatsPlugin*)h;
    if (p->hub) p->hub->leave (p->slot);
    else { b200m_bim_destroy (p->bim); b200m_sdh_destroy (p->sdh); }
    p->stage.release ();
    delete p;
}

// state extension: bitmeter -> "bim_state" = averaging (:352-388); SigDistHist -> "sdh_state" = ui_settings | ftm << 8 (:391-433)
uint32_t stats_save (LV2_Handle h, LV2_State_Store_Function store, void* handle, uint32_t, const LV2_Feature* const*)
{
    StatsPlugin* p = (StatsPlugin*)h;
    const uint32_t cfg = p->is_bim ? (p->averaging ? 1u : 0u) : (p->ui_settings | (uint32_t)p->follow_transport_mode << 8);
    store (handle, p->is_bim ? p->u.bim_state : p->u.sdh_state, &cfg, sizeof (uint32_t), p->u.atom_Int, 1u | 2u);
    return 0;
}

uint32_t stats_restore (LV2_Handle h, LV2_State_Retrieve_Function retrieve, void* handle, uint32_t, const LV2_Feature* const*)
{
    StatsPlugin* p = (StatsPlugin*)h;
    size_t size = 0; uint32_t type = 0, vflags = 0;
    const void* value = retrieve (handle, p->is_bim ? p->u.bim_state : p->u.sdh_state, &size, &type, &vflags);
    if (value && size == sizeof (uint32_t) && type == p->u.atom_Int) {
        const uint32_t cfg = *(const uint32_t*)value;
        if (p->is_bim) { p->averaging = (cfg & 1u) != 0; p->mode_dirty = true; }
        else { p->ui_settings = cfg & 0xff; p->follow_transport_mode = (cfg >> 8) & 0x3; }
        p->send_state_to_ui = true;
    }
    return 0;
}

const void* stats_extension_data (const char* uri)
{
    static const LV2_State_Interface state = {stats_save, stats_restore};
    return strcmp (uri, B200M_LV2_STATE_INTERFACE) ? nullptr : &state;
}

const LV2_Descriptor g_sdh = {MTR_URI "SigDistHist", stats_instantiate, stats_connect, nullptr, stats_run, nullptr, stats_cleanup, stats_extension_data};
const LV2_Descriptor g_bim = {MTR_URI "bitmeter", stats_instantiate, stats_connect, nullptr, stats_run, nullptr, stats_cleanup, stats_extension_data};

}  // namespace

namespace b200m {
const LV2_Descriptor* lv2_sigdisthist_descriptor () { return &g_sdh; }
const LV2_Descriptor* lv2_bitmeter_descriptor () { return &g_bim; }
}
