// lv2_xfer.cu — the "phasewheel" and "stereoscope" plugins (descriptors 23, 24 of the reference, src/meters.cc:769-770):
// xfer_run (src/xfer.c:180-276) forwards the raw stereo block to the GUI as one rawstereo object (two atom:Vector of
// float) while the UI is open, answers ui_on with a ui_state {samplerate} message, and -- phasewheel only -- runs the
// stereo correlation meter whose value goes to control port 6.  The correlation runs on the GPU (b200m_cor_*); the FFT
// analysis the reference's GUI performs on the forwarded audio is available GPU-side through b200m_pw_* (pw.cu).
// Batched mode (B200M_LV2_BATCH): a phasewheel takes a slot in the COR plugin's hub of its sample rate (cor_hub_cycle,
// lv2_shim.cu); its phase port gets the previous cycle's reading, and a skipped cycle is held in the bank.  The notify messages
// and the audio stay in their own cycle.  The stereoscope has no DSP and no bank.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "lv2_hub.cuh"

namespace {

using namespace b200m;

enum { SPR_CONTROL = 0, SPR_NOTIFY, SPR_INPUT0, SPR_OUTPUT0, SPR_INPUT1, SPR_OUTPUT1, SPR_PHASE, SPR_GAIN, SPR_RANGE };

struct XferPlugin {
    b200m_cor* cor = nullptr;                                  // phasewheel only (:93-95)
    SlotHub* hub = nullptr; int slot = -1;                     // batched phasewheel: a slot of the COR hub instead of `cor`
    bool last_ran = false;                                     // batched: the previous run() metered its cycle
    PinnedStage stage;
    AtomWriter out;
    const void* control = nullptr; void* notify = nullptr;
    float* input[2] = {nullptr, nullptr}; float* output[2] = {nullptr, nullptr}; float* p_phase = nullptr;
    double rate = 48000; bool ui_active = false, send_settings_to_ui = false, warned = false;
    LV2_URID atom_Blank = 0, atom_Object = 0, rawstereo = 0, audioleft = 0, audioright = 0, samplerate = 0, ui_on = 0, ui_off = 0, ui_state = 0;
};

LV2_Handle xfer_instantiate (const LV2_Descriptor* d, double rate, const char*, const LV2_Feature* const* features)
{
    const LV2_URID_Map* map = find_urid_map (features);
    if (!map) { fprintf (stderr, "meters.lv2 error: Host does not support urid:map\n"); return nullptr; }
    const bool wheel = !strcmp (d->URI, MTR_URI "phasewheel");
    if (!wheel && strcmp (d->URI, MTR_URI "stereoscope")) return nullptr;
    XferPlugin* p = new (std::nothrow) XferPlugin;
    if (!p) return nullptr;
    if (wheel) p->hub = cor_hub_join (rate, p, &p->slot);
    if (wheel && !p->hub && b200m_cor_create (&p->cor, 0, 1, (int)rate, 2e3f, 0.3f)) { delete p; return nullptr; }
    p->rate = rate;
    auto M = [&] (const char* uri) { return map->map (map->handle, uri); };
    p->atom_Blank = M (B200M_LV2_ATOM "Blank"); p->atom_Object = M (B200M_LV2_ATOM "Object");
    p->out.t_sequence = M (B200M_LV2_ATOM "Sequence"); p->out.t_object = p->atom_Object; p->out.t_vector = M (B200M_LV2_ATOM "Vector");
    p->out.t_float = M (B200M_LV2_ATOM "Float"); p->out.t_int = M (B200M_LV2_ATOM "Int");
    p->rawstereo = M (MTR_URI "rawstereo"); p->audioleft = M (MTR_URI "audioleft"); p->audioright = M (MTR_URI "audioright");
    p->samplerate = M (MTR_URI "samplerate"); p->ui_on = M (MTR_URI "ui_on"); p->ui_off = M (MTR_URI "ui_off"); p->ui_state = M (MTR_URI "ui_state");
    if (p->cor) p->stage.reserve (2);
    return p;
}

void xfer_connect (LV2_Handle h, uint32_t port, void* data)
{
    XferPlugin* p = (XferPlugin*)h;
    switch (port) {
    case SPR_CONTROL: p->control = data; break;
    case SPR_NOTIFY: p->notify = data; break;
    case SPR_INPUT0: p->input[0] = (float*)data; break;
    case SPR_OUTPUT0: p->output[0] = (float*)data; break;
    case SPR_INPUT1: p->input[1] = (float*)data; break;
    case SPR_OUTPUT1: p->output[1] = (float*)data; break;
    case SPR_PHASE: p->p_phase = (float*)data; break;
    default: break;
    }
}

// stcor->process; *p_phase = stcor->read () (:248-251).  Batched: the phase port gets the reading of the previous cycle unless
// that one was skipped, and a skipped cycle (atom buffer too small: no process () in the reference) is submitted held.
void xfer_meter (XferPlugin* p, uint32_t n, bool skipped)
{
    if (n < 1 || n > B200M_MAX_BLOCK) { p->last_ran = false; return; }
    if (p->hub) {
        const float v = cor_hub_cycle (p->hub, p->slot, p->input, n, skipped);
        if (p->last_ran && p->p_phase) *p->p_phase = v;
        p->last_ran = !skipped;
    } else if (p->cor && !skipped && p->stage.fill (p->input, 2, n)) {
        float v = 0;
        if (b200m_cor_process_host (p->cor, p->stage.data, p->stage.cap, n) == 0 && b200m_cor_results (p->cor, &v, nullptr) == 0 && p->p_phase) *p->p_phase = v;
    }
}

void xfer_run (LV2_Handle h, uint32_t n)
{
    XferPlugin* p = (XferPlugin*)h;
    // audio first: the reference forwards it at the end of xfer_run (src/xfer.c:262-275) and therefore DROPS it in a cycle whose
    // atom buffer is too small (:192-205); here a metering / messaging problem never costs audio
    forward_audio (p->input, p->output, 2, n);
    if (!p->notify || !p->input[0] || !p->input[1]) return;
    const size_t size = (sizeof (float) * n + 64) * 2;
    const uint32_t capacity = ((const AtomHead*)p->notify)->size;
    if (capacity < size + 128) {                               // the whole cycle is skipped, as in the reference (:190-205)
        if (!p->warned) { fprintf (stderr, "meters.lv2 error: LV2 comm-buffersize is insufficient %u/%zu bytes.\n", capacity, size + 160); p->warned = true; }
        xfer_meter (p, n, true);
        return;
    }
    p->out.begin_sequence (p->notify, capacity);
    if (p->send_settings_to_ui && p->ui_active) {
        p->send_settings_to_ui = false;
        p->out.begin_event_object (p->ui_state);
        p->out.prop_float (p->samplerate, (float)p->rate);
        p->out.end_object ();
    }
    if (p->control) {
        for (AtomEvents ev (p->control); ev.valid (); ev.next ()) {
            const AtomHead* a = ev.body ();
            if (a->type != p->atom_Blank && a->type != p->atom_Object) continue;
            AtomObject obj; obj.a = a;
            if (obj.otype () == p->ui_on) { p->ui_active = true; p->send_settings_to_ui = true; }
            else if (obj.otype () == p->ui_off) p->ui_active = false;
        }
    }
    xfer_meter (p, n, false);
    if (p->ui_active) {                                        // tx_rawstereo (:162-178)
        p->out.begin_event_object (p->rawstereo);
        p->out.prop_vector_f32 (p->audioleft, p->input[0], n);
        p->out.prop_vector_f32 (p->audioright, p->input[1], n);
        p->out.end_object ();
    }
}

void xfer_cleanup (LV2_Handle h)
{
    XferPlugin* p = (XferPlugin*)h;
    if (p->hub) p->hub->leave (p->slot);
    b200m_cor_destroy (p->cor);
    p->stage.release ();
    delete p;
}

const void* xfer_extension_data (const char*) { return nullptr; }

const LV2_Descriptor g_wheel = {MTR_URI "phasewheel", xfer_instantiate, xfer_connect, nullptr, xfer_run, nullptr, xfer_cleanup, xfer_extension_data};
const LV2_Descriptor g_scope = {MTR_URI "stereoscope", xfer_instantiate, xfer_connect, nullptr, xfer_run, nullptr, xfer_cleanup, xfer_extension_data};

}  // namespace

namespace b200m { const LV2_Descriptor* lv2_xfer_descriptor (uint32_t i) { return i == 0 ? &g_wheel : i == 1 ? &g_scope : nullptr; } }
