// lv2_gon.cu — the goniometer plugin of the LV2 façade (the 38th descriptor of src/meters.cc:745-792).
//
// Replaces goniometer_instantiate / _run / _save / _restore (src/goniometerlv2.c:44-330).  The plugin's DSP is one Stcorrdsp
// (stereo correlation, b200m_cor_*); everything else is the feed for its GUI: while the GUI is open, run() appends the block to
// a lock-free stereo ring buffer and counts a redraw notification every rate / 25 samples (:144-186).
//
// The reference GUI does not talk to the plugin through ports alone: it takes the LV2 instance handle through instance-access
// and reads / writes the plugin's C struct directly (gui/goniometer.c: self->rb, ui_active, rb_overrun, the s_* settings, the
// redraw lock).  To be a drop-in for that GUI the handle returned here points at a struct whose leading part is laid out
// exactly like `LV2gm` (src/goniometer.h:113-169, restated below member for member; x86-64 SysV layout) and whose ring buffer
// is a `gmringbuf` (:33-39) with the reference's index discipline (:52-113); this library's own state follows after it.
// tests/test_lv2_gon_gpu.py drives both plugins side by side through that struct, the way the GUI does.
// Batched mode (B200M_LV2_BATCH): the instance takes a slot in the COR plugin's hub of its sample rate (cor_hub_cycle,
// lv2_shim.cu).  The ring buffer, its overrun flag and the redraw notification stay on the host in their own cycle; the
// correlation port of run k + 1 gets cycle k's reading if the GUI was open (ui_active) in run k, the reference's rule one cycle late.
#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include "lv2_hub.cuh"

namespace {

using namespace b200m;

struct GmRing { float* c0; float* c1; size_t rp, wp, len; };                  // gmringbuf, src/goniometer.h:33-39

struct LV2gmLayout {                                                          // LV2gm, src/goniometer.h:113-169
    /* shared with ui */
    GmRing* rb; bool ui_active; bool rb_overrun;
    /* ui state/settings */
    volatile bool s_autogain, s_oversample, s_line, s_persist, s_preferences;
    volatile int s_sfact;
    volatile float s_linewidth, s_pointwidth, s_persistency, s_max_freq, s_compress, s_gattack, s_gdecay, s_gtarget, s_grms;
    /* private */
    float* input[2]; float* output[2];
    float* gain; float* notify; float* correlation;
    double rate;
    uint32_t ntfy, apv, sample_cnt;
    void* cor;                                                                // Stcorrdsp* in the reference: unused here
    /* explicit thread/redraw sync */
    pthread_mutex_t* msg_thread_lock; pthread_cond_t* data_ready; void (*queue_display) (void*); void* ui;
    /* URI */
    LV2_URID_Map* map;
    LV2_URID atom_Vector, atom_Int, atom_Float, gon_State_F, gon_State_I;
};

struct GonPlugin {
    LV2gmLayout g;                          // MUST stay first: the GUI casts the instance handle to LV2gm*
    b200m_cor* bank = nullptr;
    PinnedStage stage;
    SlotHub* hub; int slot;                 // batched: a slot of the COR hub instead of `bank`
    bool last_ui;                           // batched: ui_active in the previous run(), which publishes its reading now
};

size_t ring_write_space (const GmRing* rb) { return rb->rp == rb->wp ? rb->len - 1 : ((rb->len + rb->rp - rb->wp) % rb->len) - 1; }   // :52-55

int ring_write (GmRing* rb, const float* c0, const float* c1, size_t len)     // gmrb_write :92-109
{
    if (ring_write_space (rb) < len) return -1;
    if (rb->wp + len <= rb->len) {
        memcpy (&rb->c0[rb->wp], c0, len * sizeof (float)); memcpy (&rb->c1[rb->wp], c1, len * sizeof (float));
    } else {
        const size_t part = rb->len - rb->wp, remn = len - part;
        memcpy (&rb->c0[rb->wp], c0, part * sizeof (float)); memcpy (&rb->c1[rb->wp], c1, part * sizeof (float));
        memcpy (rb->c0, &c0[part], remn * sizeof (float)); memcpy (rb->c1, &c1[part], remn * sizeof (float));
    }
    rb->wp = (rb->wp + len) % rb->len;
    return 0;
}

LV2_Handle gon_instantiate (const LV2_Descriptor*, double rate, const char*, const LV2_Feature* const* features)
{
    LV2_URID_Map* map = find_urid_map (features);
    if (!map) { fprintf (stderr, "Goniometer error: Host does not support urid:map\n"); return nullptr; }      // :60-64
    GonPlugin* p = (GonPlugin*)calloc (1, sizeof (GonPlugin));
    if (!p) return nullptr;
    LV2gmLayout& g = p->g;
    g.map = map;
    g.atom_Vector = map->map (map->handle, B200M_LV2_ATOM "Vector");
    g.atom_Int = map->map (map->handle, B200M_LV2_ATOM "Int");
    g.atom_Float = map->map (map->handle, B200M_LV2_ATOM "Float");
    g.gon_State_F = map->map (map->handle, MTR_URI "gon_stateF");
    g.gon_State_I = map->map (map->handle, MTR_URI "gon_stateI");
    p->hub = cor_hub_join (rate, p, &p->slot);
    if (!p->hub && b200m_cor_create (&p->bank, 0, 1, (int)rate, 2e3f, 0.3f)) { free (p); return nullptr; }    // cor->init (rate, 2e3f, 0.3f) :73-74
    g.rate = rate; g.ui_active = false; g.rb_overrun = false;
    g.apv = (uint32_t)rint (rate / 25.0);                                      // UPDATE_FPS :25,80
    g.sample_cnt = 0; g.ntfy = 0;
    g.s_autogain = false; g.s_oversample = false; g.s_line = false; g.s_persist = false; g.s_preferences = false;
    g.s_sfact = 4; g.s_linewidth = .75; g.s_pointwidth = 1.75; g.s_persistency = 33; g.s_max_freq = 50;     // :89-104
    g.s_compress = 0.0; g.s_gattack = 54.0; g.s_gdecay = 58.0; g.s_gtarget = 40.0; g.s_grms = 50.0;
    uint32_t rbsize = (uint32_t)(rate / 5);                                    // :106-110
    if (rbsize < 8192u) rbsize = 8192u;
    if (rbsize < 2 * g.apv) rbsize = 2 * g.apv;
    GmRing* rb = (GmRing*)malloc (sizeof (GmRing));                            // gmrb_alloc :41-49 (plain malloc: the GUI never frees it)
    if (rb) { rb->c0 = (float*)malloc (rbsize * sizeof (float)); rb->c1 = (float*)malloc (rbsize * sizeof (float)); rb->len = rbsize; rb->rp = 0; rb->wp = 0; }
    if (!rb || !rb->c0 || !rb->c1) {
        if (rb) { free (rb->c0); free (rb->c1); free (rb); }
        if (p->hub) p->hub->leave (p->slot);
        b200m_cor_destroy (p->bank); free (p); return nullptr;
    }
    g.rb = rb;
    if (!p->hub) p->stage.reserve (2);
    return p;
}

void gon_connect (LV2_Handle h, uint32_t port, void* data)                    // JFPortIndex :27-35
{
    LV2gmLayout& g = ((GonPlugin*)h)->g;
    switch (port) {
    case 0: g.input[0] = (float*)data; break;
    case 1: g.output[0] = (float*)data; break;
    case 2: g.input[1] = (float*)data; break;
    case 3: g.output[1] = (float*)data; break;
    case 4: g.gain = (float*)data; break;
    case 5: g.correlation = (float*)data; break;
    case 6: g.notify = (float*)data; break;
    default: break;
    }
}

void gon_run (LV2_Handle h, uint32_t n)
{
    GonPlugin* p = (GonPlugin*)h; LV2gmLayout& g = p->g;
    // audio first: a metering failure never drops it (the reference copies last, :177-182)
    forward_audio (g.input, g.output, 2, n);
    if (!g.input[0] || !g.input[1] || n == 0) return;
    // self->cor->process (in0, in1, n) every cycle, GUI open or not (:147); cycles longer than the engine's block go in pieces
    bool ok = true; float cv = 0;
    for (uint32_t off = 0; off < n && ok; off += B200M_MAX_BLOCK) {
        const uint32_t k = n - off < B200M_MAX_BLOCK ? n - off : B200M_MAX_BLOCK;
        const float* in[2] = {g.input[0] + off, g.input[1] + off};
        if (p->hub) { cv = cor_hub_cycle (p->hub, p->slot, in, k, false); continue; }
        ok = p->stage.fill (in, 2, k) && b200m_cor_process_host (p->bank, p->stage.data, p->stage.cap, k) == 0;
        if (ok && off + k < n) { float tmp; ok = b200m_cor_results (p->bank, &tmp, nullptr) == 0; }      // `stage` is reused by the next piece: wait for its upload
    }
    // cor->read () reaches the port while the GUI is open (:174); batched: the previous cycle's reading, if the GUI was open in
    // that cycle.  Private: the results call is also the stream sync (`stage` is free when run() returns)
    const bool ui = g.ui_active;
    const bool show = p->hub ? p->last_ui : ok && b200m_cor_results (p->bank, &cv, nullptr) == 0 && ui;
    p->last_ui = ui;
    if (g.correlation && show) *g.correlation = cv;
    if (ui) {
        if (ring_write (g.rb, g.input[0], g.input[1], n) < 0) g.rb_overrun = true;                    // reset by UI (:150-152)
        g.sample_cnt += n;                                                     // notify UI about new data (:155-172)
        if (g.sample_cnt >= g.apv) {
            if (g.msg_thread_lock) {
                g.queue_display (g.ui);
                if (pthread_mutex_trylock (g.msg_thread_lock) == 0) { pthread_cond_signal (g.data_ready); pthread_mutex_unlock (g.msg_thread_lock); }
            } else g.ntfy = (g.ntfy + 1) % 10000;
            g.sample_cnt = g.sample_cnt % g.apv;
        }
        if (g.notify) *g.notify = (float)g.ntfy;
    } else g.rb_overrun = false;
}

void gon_cleanup (LV2_Handle h)
{
    GonPlugin* p = (GonPlugin*)h;
    if (p->hub) p->hub->leave (p->slot);
    free (p->g.rb->c0); free (p->g.rb->c1); free (p->g.rb);
    b200m_cor_destroy (p->bank);
    p->stage.release ();
    free (p);
}

struct VectorOfFloat { uint32_t child_size, child_type; float cfg[9]; };     // :197-207
struct VectorOfInt { uint32_t child_size, child_type; int32_t cfg[2]; };

uint32_t gon_save (LV2_Handle h, LV2_State_Store_Function store, void* handle, uint32_t, const LV2_Feature* const*)       // :209-253
{
    LV2gmLayout& g = ((GonPlugin*)h)->g;
    VectorOfFloat vof; VectorOfInt voi;
    vof.child_type = g.atom_Float; vof.child_size = sizeof (float);
    voi.child_type = g.atom_Int; voi.child_size = sizeof (int32_t);
    vof.cfg[0] = g.s_linewidth; vof.cfg[1] = g.s_pointwidth; vof.cfg[2] = g.s_persistency; vof.cfg[3] = g.s_max_freq; vof.cfg[4] = g.s_compress;
    vof.cfg[5] = g.s_gattack; vof.cfg[6] = g.s_gdecay; vof.cfg[7] = g.s_gtarget; vof.cfg[8] = g.s_grms;
    voi.cfg[1] = g.s_sfact;
    voi.cfg[0] = (g.s_autogain ? 1 : 0) | (g.s_oversample ? 2 : 0) | (g.s_line ? 4 : 0) | (g.s_persist ? 8 : 0) | (g.s_preferences ? 16 : 0);
    store (handle, g.gon_State_F, &vof, sizeof (vof), g.atom_Vector, 1u /* LV2_STATE_IS_POD */);
    store (handle, g.gon_State_I, &voi, sizeof (voi), g.atom_Vector, 1u);
    return 0;
}

uint32_t gon_restore (LV2_Handle h, LV2_State_Retrieve_Function retrieve, void* handle, uint32_t, const LV2_Feature* const*)   // :255-294
{
    LV2gmLayout& g = ((GonPlugin*)h)->g;
    size_t size = 0; uint32_t type = 0, vflags = 0;
    const void* v1 = retrieve (handle, g.gon_State_F, &size, &type, &vflags);
    if (v1 && size == 8 + 9 * sizeof (float) && type == g.atom_Vector) {
        const float* cfg = (const float*)((const uint8_t*)v1 + 8);              // LV2_ATOM_BODY: past the vector body head {child_size, child_type}
        g.s_linewidth = cfg[0]; g.s_pointwidth = cfg[1]; g.s_persistency = cfg[2]; g.s_max_freq = cfg[3]; g.s_compress = cfg[4];
        g.s_gattack = cfg[5]; g.s_gdecay = cfg[6]; g.s_gtarget = cfg[7]; g.s_grms = cfg[8];
    }
    const void* v2 = retrieve (handle, g.gon_State_I, &size, &type, &vflags);
    if (v2 && size == 8 + 2 * sizeof (int32_t) && type == g.atom_Vector) {
        const int32_t* cfg = (const int32_t*)((const uint8_t*)v2 + 8);
        g.s_sfact = cfg[1];
        g.s_autogain = (cfg[0] & 1) != 0; g.s_oversample = (cfg[0] & 2) != 0; g.s_line = (cfg[0] & 4) != 0;
        g.s_persist = (cfg[0] & 8) != 0; g.s_preferences = (cfg[0] & 16) != 0;
    }
    return 0;
}

const void* gon_extension_data (const char* uri)
{
    static const LV2_State_Interface state = {gon_save, gon_restore};
    return strcmp (uri, B200M_LV2_STATE_INTERFACE) ? nullptr : &state;
}

const LV2_Descriptor g_gon = {MTR_URI "goniometer", gon_instantiate, gon_connect, nullptr, gon_run, nullptr, gon_cleanup, gon_extension_data};

}  // namespace

namespace b200m { const LV2_Descriptor* lv2_goniometer_descriptor () { return &g_gon; } }

// layout of the GUI-shared part, for tests: offsets of rb, ui_active, rb_overrun, s_sfact, s_linewidth, input, rate, ntfy, msg_thread_lock, map, sizeof
extern "C" int b200m_lv2_gon_layout (size_t* out, int n)
{
    const size_t v[] = {offsetof (LV2gmLayout, rb), offsetof (LV2gmLayout, ui_active), offsetof (LV2gmLayout, rb_overrun), offsetof (LV2gmLayout, s_sfact),
                        offsetof (LV2gmLayout, s_linewidth), offsetof (LV2gmLayout, input), offsetof (LV2gmLayout, rate), offsetof (LV2gmLayout, ntfy),
                        offsetof (LV2gmLayout, msg_thread_lock), offsetof (LV2gmLayout, map), sizeof (LV2gmLayout)};
    const int m = (int)(sizeof (v) / sizeof (v[0]));
    for (int i = 0; i < n && i < m; ++i) out[i] = v[i];
    return m;
}
