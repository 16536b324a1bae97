/* lv2_host.c — a minimal LV2 host for throughput measurements of the plugin façade (plain C, no LV2 SDK).
 *
 * Does what robtk/jackwrap.c:531-544 does once per audio period — connect ports, run() every instance — for N instances of ONE
 * plugin URI loaded from an LV2 binary (libb200meters.so, or the reference's meters.so), and times the cycle:
 *
 *     lv2_host --lib meters.lv2_b200/libb200meters.so --uri EBUr128 --instances 8192 --cycles 200 [--nframes 1024]
 *              [--rate 48000] [--ui 0|1] [--threads 1]
 *
 * prints one JSON line: mean / max cycle time, microseconds per instance and cycle, the real-time budget nframes / rate and whether
 * the cycle fits in it.  With B200M_LV2_BATCH=<slots> in the environment the façade's instances share banks (one upload and one
 * set of kernel launches per cycle for all of them); without it every instance is a synchronous bank of one.
 *
 * Port layouts (restated from the reference's TTL / port enums):
 *   EBUr128 (src/ebulv2.cc:31-38): 0 control atom in, 1 notify atom out, 2 inL, 3 outL, 4 inR, 5 outR
 *   needle / COR / dBTP / K-meters (src/meters.cc:59-70): 0 reflevel, 1 in0, 2 out0, 3 level0, 4 in1, 5 out1, 6 level1, 7 peak0, 8 peak1, 9 hold
 *   spectr30 (src/spectrumlv2.c:35-44): 0-59 band / max outputs, 60 speed, 61 reset, 62 amp, 63 state, 64 in0, 65 out0, 66 in1, 67 out1
 *   bitmeter / SigDistHist (src/bitmeter.c, src/sigdistlv2.c port enums): 0 control atom in, 1 notify atom out, 2 in, 3 out
 *   dr14mono/stereo, TPnRMSmono/stereo (src/dr14.c:27-43): 0 control atom in, 1 follow host transport, 2 reset, 3 block count,
 *                4 in0, 5 out0, 6-10 outputs of channel 0, 11 in1, 12 out1, 13-17 outputs of channel 1, 18 DR total (no notify port)
 *   surround3..8 (src/surmeter.c:24-70): pair c: 1 + 3c, 2 + 3c input selectors, 3 + 3c correlation; channel c: 13 + 4c in, 14 + 4c out,
 *                15 + 4c level, 16 + 4c peak
 *   phasewheel / stereoscope (src/xfer.c:50-60): 0 control atom in, 1 notify atom out, 2 in0, 3 out0, 4 in1, 5 out1, 6 phase, 7 gain, 8 range;
 *                the notify buffer holds one rawstereo message of both channels per cycle, (4 n + 64) * 2 + 128 bytes (:188-205)
 *   goniometer (src/goniometerlv2.c:27-35): 0 in0, 1 out0, 2 in1, 3 out1, 4 gain, 5 correlation, 6 notify
 * --ui 1 opens the GUI: meteron (EBUr128, bitmeter, SigDistHist), ui_on (phasewheel, stereoscope); the goniometer's GUI sets ui_active
 * in the plugin's instance struct (LV2gm, src/goniometer.h:113-169) and drains its ring buffer every cycle, which this host does too.
 */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

typedef void* LV2_Handle;
typedef struct { const char* URI; void* data; } LV2_Feature;
typedef struct LV2_Descriptor_s {
    const char* URI;
    LV2_Handle (*instantiate) (const struct LV2_Descriptor_s*, double, const char*, const LV2_Feature* const*);
    void (*connect_port) (LV2_Handle, uint32_t, void*);
    void (*activate) (LV2_Handle);
    void (*run) (LV2_Handle, uint32_t);
    void (*deactivate) (LV2_Handle);
    void (*cleanup) (LV2_Handle);
    const void* (*extension_data) (const char*);
} LV2_Descriptor;
typedef struct { void* handle; uint32_t (*map) (void*, const char*); } LV2_URID_Map;

#define MTR_URI "http://gareus.org/oss/lv2/meters#"
#define MAXURI 256
static char* g_uri[MAXURI]; static int g_nuri = 0; static pthread_mutex_t g_mu = PTHREAD_MUTEX_INITIALIZER;
static uint32_t urid_map (void* h, const char* uri)
{
    (void)h;
    pthread_mutex_lock (&g_mu);
    int i;
    for (i = 0; i < g_nuri; ++i) if (!strcmp (g_uri[i], uri)) break;
    if (i == g_nuri && g_nuri < MAXURI) g_uri[g_nuri++] = strdup (uri);
    pthread_mutex_unlock (&g_mu);
    return (uint32_t)i + 1;
}

typedef struct {
    LV2_Handle h;
    float *in[8], *out[8];
    float ctl[68];                          /* control ports (in and out) */
    uint8_t *atom_in, *atom_out;            /* EBUr128, bitmeter, SigDistHist, phasewheel, stereoscope */
} Inst;

typedef struct { const LV2_Descriptor* d; Inst* inst; int first, last; uint32_t nframes; int kind; uint32_t seq_t, chunk_t, atom_cap; pthread_barrier_t *start, *done;
                 int cycles; int cycle; const uint8_t* first_msgs; uint32_t first_len; int ui; } Worker;

enum { KIND_MTR, KIND_EBUR, KIND_SPEC, KIND_STATS, KIND_SUR, KIND_DR, KIND_XFER, KIND_GON };
#define ATOM_CAP 8192
/* goniometer: the GUI-shared head of LV2gm (src/goniometer.h:33-39,113-116): gmringbuf* rb, then bool ui_active; the ring is
 * {float* c0, c1; size_t rp, wp, len} */
typedef struct { float *c0, *c1; size_t rp, wp, len; } GmRing;
typedef struct { GmRing* rb; _Bool ui_active; } GmHead;

/* one event at frame 0: object {otype; controlkey = key (Int); controlval = val (Float)} -- forge_kvcontrolmessage, src/uris.h:279-294 */
static uint32_t forge_kv (uint8_t* dst, uint32_t t_object, uint32_t otype, uint32_t t_int, uint32_t t_float, uint32_t k_key, uint32_t k_val, int key, float val, int with_props)
{
    uint32_t w[18]; memset (w, 0, sizeof (w));
    const uint32_t body = with_props ? 8 + 48 : 8;
    w[0] = 0; w[1] = 0;                                  /* int64 frames */
    w[2] = body; w[3] = t_object; w[4] = 1; w[5] = otype;
    if (with_props) {
        w[6] = k_key; w[7] = 0; w[8] = 4; w[9] = t_int; memcpy (&w[10], &key, 4);
        w[12] = k_val; w[13] = 0; w[14] = 4; w[15] = t_float; memcpy (&w[16], &val, 4);
    }
    const uint32_t n = 16 + body;
    memcpy (dst, w, n);
    return n;
}

static double now_s (void) { struct timespec ts; clock_gettime (CLOCK_MONOTONIC, &ts); return ts.tv_sec + 1e-9 * ts.tv_nsec; }

static void run_range (const Worker* w)
{
    for (int i = w->first; i < w->last; ++i) {
        Inst* p = &w->inst[i];
        if (w->kind == KIND_DR) { uint32_t* a = (uint32_t*)p->atom_in; a[0] = 8; a[1] = w->seq_t; a[2] = 0; a[3] = 0; }   /* empty input sequence */
        if (w->kind == KIND_EBUR || w->kind == KIND_STATS || w->kind == KIND_XFER) {   /* host convention: empty input sequence, output buffer announced as a chunk of its capacity */
            uint32_t* a = (uint32_t*)p->atom_in; a[0] = 8; a[1] = w->seq_t; a[2] = 0; a[3] = 0;
            if (w->cycle == 0 && w->first_len) { memcpy (p->atom_in + 16, w->first_msgs, w->first_len); a[0] = 8 + w->first_len; }   /* the GUI's opening messages */
            uint32_t* o = (uint32_t*)p->atom_out; o[0] = w->atom_cap - 8; o[1] = w->chunk_t;
        }
        if (w->kind == KIND_GON && w->ui) { GmHead* g = (GmHead*)p->h; g->ui_active = 1; g->rb->rp = g->rb->wp; }   /* the GUI's open / gmrb_read_clear */
        w->d->run (p->h, w->nframes);
    }
}

static void* worker_main (void* arg)
{
    Worker* w = (Worker*)arg;
    for (int c = 0; c < w->cycles; ++c) {
        pthread_barrier_wait (w->start);
        w->cycle = c;
        run_range (w);
        pthread_barrier_wait (w->done);
    }
    return NULL;
}

int main (int argc, char** argv)
{
    const char* lib = "meters.lv2_b200/libb200meters.so"; const char* uri = "EBUr128";
    int n_inst = 256, cycles = 100, threads = 1, warm = 5, dbtp = 1, ui = 0; uint32_t nframes = 1024; double rate = 48000.0;
    for (int i = 1; i + 1 < argc; i += 2) {
        if (!strcmp (argv[i], "--lib")) lib = argv[i + 1];
        else if (!strcmp (argv[i], "--uri")) uri = argv[i + 1];
        else if (!strcmp (argv[i], "--instances")) n_inst = atoi (argv[i + 1]);
        else if (!strcmp (argv[i], "--cycles")) cycles = atoi (argv[i + 1]);
        else if (!strcmp (argv[i], "--warmup")) warm = atoi (argv[i + 1]);
        else if (!strcmp (argv[i], "--nframes")) nframes = (uint32_t)atoi (argv[i + 1]);
        else if (!strcmp (argv[i], "--rate")) rate = atof (argv[i + 1]);
        else if (!strcmp (argv[i], "--threads")) threads = atoi (argv[i + 1]);
        else if (!strcmp (argv[i], "--dbtp")) dbtp = atoi (argv[i + 1]);       /* EBUr128: enable the true-peak meters (CTL_UISETTINGS bit 64) */
        else if (!strcmp (argv[i], "--ui")) ui = atoi (argv[i + 1]);           /* a GUI is attached (EBUr128, bitmeter, SigDistHist, phasewheel, stereoscope, goniometer) */
        else { fprintf (stderr, "unknown option %s\n", argv[i]); return 2; }
    }
    if (threads < 1) threads = 1;
    if (threads > n_inst) threads = n_inst;
    void* so = dlopen (lib, RTLD_NOW | RTLD_LOCAL);
    if (!so) { fprintf (stderr, "dlopen: %s\n", dlerror ()); return 1; }
    const LV2_Descriptor* (*get) (uint32_t) = (const LV2_Descriptor* (*) (uint32_t))dlsym (so, "lv2_descriptor");
    if (!get) { fprintf (stderr, "no lv2_descriptor in %s\n", lib); return 1; }
    char full[512]; snprintf (full, sizeof (full), MTR_URI "%s", uri);
    const LV2_Descriptor* d = NULL;
    for (uint32_t i = 0; (d = get (i)) != NULL; ++i) if (!strcmp (d->URI, full)) break;
    if (!d) { fprintf (stderr, "%s not served by %s\n", full, lib); return 1; }
    const int kind = !strcmp (uri, "EBUr128") ? KIND_EBUR : !strncmp (uri, "spectr30", 8) ? KIND_SPEC
                   : !strcmp (uri, "bitmeter") || !strcmp (uri, "SigDistHist") ? KIND_STATS : !strncmp (uri, "surround", 8) ? KIND_SUR
                   : !strncmp (uri, "dr14", 4) || !strncmp (uri, "TPnRMS", 6) ? KIND_DR
                   : !strcmp (uri, "phasewheel") || !strcmp (uri, "stereoscope") ? KIND_XFER : !strcmp (uri, "goniometer") ? KIND_GON : KIND_MTR;
    const int stereo = kind == KIND_EBUR || kind == KIND_XFER || kind == KIND_GON || strstr (uri, "stereo") || !strcmp (uri, "COR") || !strcmp (uri, "BBCM6");
    const uint32_t atom_cap = kind == KIND_XFER ? (4 * nframes + 64) * 2 + 1024 : ATOM_CAP;
    const int chn = kind == KIND_SUR ? uri[8] - '0' : stereo ? 2 : 1;

    LV2_URID_Map map = {NULL, urid_map};
    LV2_Feature fmap = {"http://lv2plug.in/ns/ext/urid#map", &map};
    const LV2_Feature* feats[2] = {&fmap, NULL};
    const uint32_t seq_t = urid_map (NULL, "http://lv2plug.in/ns/ext/atom#Sequence"), chunk_t = urid_map (NULL, "http://lv2plug.in/ns/ext/atom#Chunk");

    /* EBUr128: what the GUI sends when it opens -- integration on, dBTP on, optionally "meteron" (src/ebulv2.cc:258-331) */
    /* bitmeter / SigDistHist (ports 0 control, 1 notify, 2 in, 3 out): "meteron" with --ui 1, and SigDistHist's CTL_START */
    uint8_t first_msgs[512]; uint32_t first_len = 0;
    if (kind == KIND_EBUR || kind == KIND_STATS) {
        const uint32_t t_obj = urid_map (NULL, "http://lv2plug.in/ns/ext/atom#Object"), t_int = urid_map (NULL, "http://lv2plug.in/ns/ext/atom#Int"),
                       t_flt = urid_map (NULL, "http://lv2plug.in/ns/ext/atom#Float"), cfg = urid_map (NULL, MTR_URI "metercfg"),
                       kk = urid_map (NULL, MTR_URI "controlkey"), kv = urid_map (NULL, MTR_URI "controlval"), on = urid_map (NULL, MTR_URI "meteron");
        if (ui) first_len += forge_kv (first_msgs + first_len, t_obj, on, t_int, t_flt, kk, kv, 0, 0, 0);
        if (kind == KIND_EBUR) first_len += forge_kv (first_msgs + first_len, t_obj, cfg, t_int, t_flt, kk, kv, 7 /* CTL_UISETTINGS */, dbtp ? 64.0f : 0.0f, 1);
        if (kind == KIND_EBUR || !strcmp (uri, "SigDistHist")) first_len += forge_kv (first_msgs + first_len, t_obj, cfg, t_int, t_flt, kk, kv, 1 /* CTL_START */, 0.0f, 1);
    }
    if (kind == KIND_XFER && ui)                        /* phasewheel / stereoscope GUI: ui_on (gui/phasewheel.c:263-270) */
        first_len += forge_kv (first_msgs, urid_map (NULL, "http://lv2plug.in/ns/ext/atom#Object"), urid_map (NULL, MTR_URI "ui_on"), 0, 0, 0, 0, 0, 0, 0);
    Inst* inst = (Inst*)calloc ((size_t)n_inst, sizeof (Inst));
    uint64_t s = 0x42B200;
    for (int i = 0; i < n_inst; ++i) {
        Inst* p = &inst[i];
        p->h = d->instantiate (d, rate, "", feats);
        if (!p->h) { fprintf (stderr, "instantiate failed at instance %d (no GPU? B200M_LV2_BATCH smaller than --instances is fine: more hubs are made)\n", i); return 1; }
        for (int c = 0; c < chn; ++c) {
            p->in[c] = (float*)malloc (sizeof (float) * nframes); p->out[c] = (float*)malloc (sizeof (float) * nframes);
            for (uint32_t k = 0; k < nframes; ++k) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; p->in[c][k] = ((float)(s >> 40) * (1.0f / 8388608.0f) - 1.0f) * 0.25f; }
        }
        if (kind == KIND_EBUR || kind == KIND_STATS || kind == KIND_XFER) {
            p->atom_in = (uint8_t*)calloc (1, 1024); p->atom_out = (uint8_t*)calloc (1, atom_cap);
            d->connect_port (p->h, 0, p->atom_in); d->connect_port (p->h, 1, p->atom_out);
            d->connect_port (p->h, 2, p->in[0]); d->connect_port (p->h, 3, p->out[0]);
            if (stereo) { d->connect_port (p->h, 4, p->in[1]); d->connect_port (p->h, 5, p->out[1]); }
            if (kind == KIND_XFER) for (uint32_t k = 6; k < 9; ++k) d->connect_port (p->h, k, &p->ctl[k]);
        } else if (kind == KIND_GON) {
            d->connect_port (p->h, 0, p->in[0]); d->connect_port (p->h, 1, p->out[0]);
            d->connect_port (p->h, 2, p->in[1]); d->connect_port (p->h, 3, p->out[1]);
            p->ctl[4] = 1.0f;
            for (uint32_t k = 4; k < 7; ++k) d->connect_port (p->h, k, &p->ctl[k]);
        } else if (kind == KIND_SPEC) {
            for (uint32_t k = 0; k < 64; ++k) d->connect_port (p->h, k, &p->ctl[k]);
            p->ctl[60] = 1.0f; p->ctl[61] = -4.0f; p->ctl[62] = 0.0f;
            d->connect_port (p->h, 64, p->in[0]); d->connect_port (p->h, 65, p->out[0]);
            if (stereo) { d->connect_port (p->h, 66, p->in[1]); d->connect_port (p->h, 67, p->out[1]); }
        } else if (kind == KIND_DR) {
            p->atom_in = (uint8_t*)calloc (1, 1024);
            d->connect_port (p->h, 0, p->atom_in);
            for (uint32_t k = 1; k < 19; ++k) if (k != 4 && k != 5 && k != 11 && k != 12) d->connect_port (p->h, k, &p->ctl[k]);
            p->ctl[1] = 1.0f;                                   /* follow host transport (the plugin's default) */
            d->connect_port (p->h, 4, p->in[0]); d->connect_port (p->h, 5, p->out[0]);
            if (stereo) { d->connect_port (p->h, 11, p->in[1]); d->connect_port (p->h, 12, p->out[1]); }
        } else if (kind == KIND_SUR) {
            for (uint32_t k = 0; k < 13; ++k) d->connect_port (p->h, k, &p->ctl[k]);
            for (int c = 0; c < 4; ++c) { p->ctl[1 + 3 * c] = (float)c; p->ctl[2 + 3 * c] = (float)((c + 1) % chn); }   /* adjacent channel pairs */
            for (int c = 0; c < chn; ++c) {
                d->connect_port (p->h, 13 + 4 * c, p->in[c]); d->connect_port (p->h, 14 + 4 * c, p->out[c]);
                d->connect_port (p->h, 15 + 4 * c, &p->ctl[15 + 4 * c]); d->connect_port (p->h, 16 + 4 * c, &p->ctl[16 + 4 * c]);
            }
        } else {
            for (uint32_t k = 0; k < 10; ++k) d->connect_port (p->h, k, &p->ctl[k]);
            p->ctl[0] = -18.0f;
            d->connect_port (p->h, 1, p->in[0]); d->connect_port (p->h, 2, p->out[0]);
            if (stereo) { d->connect_port (p->h, 4, p->in[1]); d->connect_port (p->h, 5, p->out[1]); }
        }
        if (d->activate) d->activate (p->h);
    }

    pthread_barrier_t b_start, b_done;
    pthread_barrier_init (&b_start, NULL, (unsigned)threads + 1); pthread_barrier_init (&b_done, NULL, (unsigned)threads + 1);
    Worker* w = (Worker*)calloc ((size_t)threads, sizeof (Worker)); pthread_t* th = (pthread_t*)calloc ((size_t)threads, sizeof (pthread_t));
    for (int t = 0; t < threads; ++t) {
        w[t].d = d; w[t].inst = inst; w[t].first = (int)((long long)n_inst * t / threads); w[t].last = (int)((long long)n_inst * (t + 1) / threads);
        w[t].nframes = nframes; w[t].kind = kind; w[t].seq_t = seq_t; w[t].chunk_t = chunk_t; w[t].atom_cap = atom_cap; w[t].ui = ui; w[t].start = &b_start; w[t].done = &b_done; w[t].cycles = warm + cycles; w[t].first_msgs = first_msgs; w[t].first_len = first_len;
        pthread_create (&th[t], NULL, worker_main, &w[t]);
    }
    double sum = 0, worst = 0;
    for (int c = 0; c < warm + cycles; ++c) {
        const double t0 = now_s ();
        pthread_barrier_wait (&b_start);
        pthread_barrier_wait (&b_done);
        const double dt = now_s () - t0;
        if (c >= warm) { sum += dt; if (dt > worst) worst = dt; }
    }
    for (int t = 0; t < threads; ++t) pthread_join (th[t], NULL);
    const double mean = sum / cycles, budget = nframes / rate;
    float probe = kind == KIND_EBUR || kind == KIND_STATS ? 0.0f : inst[0].ctl[kind == KIND_DR || kind == KIND_XFER ? 6 : kind == KIND_GON ? 5 : 3];
    const char* batch = getenv ("B200M_LV2_BATCH");
    printf ("{\"lv2_host\": \"%s\", \"lib\": \"%s\", \"instances\": %d, \"threads\": %d, \"nframes\": %u, \"rate\": %.0f, \"cycles\": %d, "
            "\"dbtp\": %d, \"ui\": %d, \"batch_slots\": %s, \"cycle_ms_mean\": %.4f, \"cycle_ms_max\": %.4f, \"us_per_instance\": %.3f, \"budget_ms\": %.3f, \"fits_realtime\": %s, "
            "\"realtime_instances_at_this_rate\": %.0f, \"probe_level0\": %g}\n",
            uri, lib, n_inst, threads, nframes, rate, cycles, dbtp, ui, batch ? batch : "null", mean * 1e3, worst * 1e3, mean * 1e6 / n_inst, budget * 1e3,
            mean < budget ? "true" : "false", n_inst * budget / mean, probe);
    for (int i = 0; i < n_inst; ++i) d->cleanup (inst[i].h);
    return 0;
}
