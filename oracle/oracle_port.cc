// oracle_port.cc — CPU restatement ("port") of the reference's metering algorithms.
//
// TEST INFRASTRUCTURE ONLY (see oracle_api.h): loaded by tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference leg, never by the product.  Written from scratch as a
// plain restatement of WHAT the reference computes, each routine citing the reference file:line it
// follows (paths relative to the x42/meters.lv2 tree).  Parity pin: tests/test_oracle_port.py checks
// every routine bit-for-bit against oracle/_ref (the unmodified reference sources compiled here) and
// against the committed golden vectors in tests/golden/ (generated from oracle/_ref by
// tests/golden/make_golden.py).  The one exception is the phasewheel FFT: the reference calls FFTW3,
// which is neither vendored nor installed, so that routine restates gui/fft.c around a
// double-precision DFT and is "parity unpinned" (DESIGN.md).
//
// Build with the reference's flags (oracle/Makefile): SSE2 float arithmetic, no FMA contraction.
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <complex>
#include <functional>
#include <thread>
#include <vector>

#include "oracle_api.h"

namespace {

void par_for (int n, int nthreads, const std::function<void (int, int)>& fn)
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

inline bool fin (float v) { return std::isfinite (v); }

// =====================================================================================
// EBU R128 — ebumeter/ebu_r128_proc.cc
// =====================================================================================
struct Hist {                                   // Ebu_r128_hist, :32-150
    int bins[751]; int count, error;
    void clear () { memset (bins, 0, sizeof (bins)); count = error = 0; }
    void add (float v) {                        // addpoint :66-79
        int k = (int)floorf (10 * v + 700.5f);
        if (k < 0) return;
        if (k > 750) { k = 750; error++; }
        bins[k]++; count++;
    }
};
float g_binpow[100];                            // _bin_power, initstat :54-63
void binpow_init () { if (g_binpow[0]) return; for (int i = 0; i < 100; ++i) g_binpow[i] = powf (10.0f, i / 100.0f); }

float hist_mean (const Hist& h, int i) {        // integrate :82-102
    int j = i % 100, n = 0; float s = 0;
    while (i <= 750) {
        int k = h.bins[i++];
        n += k;
        s += k * g_binpow[j++];
        if (j == 100) { j = 0; s /= 10.0f; }
    }
    return s / n;
}
void hist_integ (const Hist& h, float* vi, float* th) {     // calc_integ :105-125
    if (h.count < 50) { *vi = -200.0f; return; }
    float s = hist_mean (h, 0);
    *th = 10 * log10f (s) - 10.0f;
    int k = (int)(floorf (100 * log10f (s) + 0.5f)) + 600;
    if (k < 0) k = 0;
    s = hist_mean (h, k);
    *vi = 10 * log10f (s);
}
void hist_range (const Hist& h, float* v0, float* v1, float* th) {   // calc_range :128-150
    if (h.count < 20) { *v0 = -200.0f; *v1 = -200.0f; return; }
    float s = hist_mean (h, 0);
    *th = 10 * log10f (s) - 20.0f;
    int k = (int)(floorf (100 * log10f (s) + 0.5)) + 500;    // 0.5 is a double literal in the reference
    if (k < 0) k = 0;
    int i, j, n;
    for (i = k, n = 0; i <= 750; i++) n += h.bins[i];
    const float a = 0.10f * n, b = 0.95f * n;
    for (i = k, s = 0; s < a; i++) s += h.bins[i];
    for (j = 750, s = n; s > b; j--) s -= h.bins[j];
    *v0 = (i - 701) / 10.0f;
    *v1 = (j - 699) / 10.0f;
}

struct Ebu {
    int nchan, fragm, frcnt, wrind, div1, div2; bool integr;
    float fsamp, frpwr, power[64];
    float lM, mM, lS, mS, integ, ithr, rmin, rmax, rthr;
    float a0, a1, a2, b1, b2, c3, c4;
    float z[5][4];
    Hist hM, hS;

    void design (float fs) {                    // detect_init :263-293 (tan of a float = float overload)
        float r = 1 / tanf (4712.3890f / fs);
        float w1 = r / 1.12201f, w2 = r * 1.12201f;
        float u = 1.4085f + 210.0f / fs;
        float a = u * w1, b = w1 * w1, c = u * w2, d = w2 * w2;
        r = 1 + a + b;
        a0 = (1 + c + d) / r; a1 = (2 - 2 * d) / r; a2 = (1 - c + d) / r;
        b1 = (2 - 2 * b) / r; b2 = (1 - a + b) / r;
        r = 48.0f / fs;
        a = 4.9886075f * r; b = 6.2298014f * r * r;
        r = 1 + a + b;
        a *= 2 / r; b *= 4 / r;
        c3 = a + b; c4 = b;
        r = 1.004995f / r;
        a0 *= r; a1 *= r; a2 *= r;
    }
    void integr_reset () {                      // :193-204
        hM.clear (); hS.clear ();
        mM = mS = integ = ithr = rmin = rmax = rthr = -200.0f;
        div1 = div2 = 0;
    }
    void reset () {                             // :176-190
        integr = false; frcnt = fragm; frpwr = 1e-30f; wrind = 0; div1 = div2 = 0;
        lM = lS = -200.0f;
        memset (power, 0, sizeof (power));
        integr_reset ();
        memset (z, 0, sizeof (z));
    }
    void init (int nc, float fs) { nchan = nc; fsamp = fs; fragm = (int)fs / 20; design (fs); binpow_init (); reset (); }

    float detect (const float* const* ip, int n) {          // detect_process :302-337
        static const float gain[5] = {1.0f, 1.0f, 1.0f, 1.41f, 1.41f};
        float si = 0;
        for (int c = 0; c < nchan; ++c) {
            float z1 = z[c][0], z2 = z[c][1], z3 = z[c][2], z4 = z[c][3], sj = 0;
            const float* p = ip[c];
            for (int j = 0; j < n; ++j) {
                float x = p[j] - b1 * z1 - b2 * z2 + 1e-15f;
                float y = a0 * x + a1 * z1 + a2 * z2 - c3 * z3 - c4 * z4;
                z2 = z1; z1 = x; z4 += z3; z3 += y;
                sj += y * y;
            }
            if (nchan == 1) si = 2 * sj; else si += gain[c] * sj;
            z[c][0] = fin (z1) ? z1 : 0; z[c][1] = fin (z2) ? z2 : 0; z[c][2] = fin (z3) ? z3 : 0; z[c][3] = fin (z4) ? z4 : 0;
        }
        return si;
    }
    float frags (int nf) {                      // addfrags :251-260
        float s = 0; int k = (wrind - nf) & 63;
        for (int i = 0; i < nf; ++i) s += power[(i + k) & 63];
        return -0.6976f + 10 * log10f (s / nf);
    }
    void process (int nfram, const float* const* in) {      // :207-248
        const float* ip[5];
        for (int c = 0; c < nchan; ++c) ip[c] = in[c];
        while (nfram) {
            int k = frcnt < nfram ? frcnt : nfram;
            frpwr += detect (ip, k);
            frcnt -= k;
            if (frcnt == 0) {
                power[wrind++] = frpwr / fragm;
                frcnt = fragm; frpwr = 1e-30f; wrind &= 63;
                lM = frags (8); lS = frags (60);
                if (!fin (lM) || lM < -200.f) lM = -200.0f;
                if (!fin (lS) || lS < -200.f) lS = -200.0f;
                if (lM > mM) mM = lM;
                if (lS > mS) mS = lS;
                if (integr) {
                    if (++div1 == 2) { hM.add (lM); div1 = 0; }
                    if (++div2 == 10) { hS.add (lS); div2 = 0; hist_integ (hM, &integ, &ithr); hist_range (hS, &rmin, &rmax, &rthr); }
                }
            }
            for (int c = 0; c < nchan; ++c) ip[c] += k;
            nfram -= k;
        }
    }
};

// =====================================================================================
// zita-resampler 1:4, hl = 24 — zita-resampler/resampler.cc, resampler-table.cc
// =====================================================================================
struct ZitaTab { float c[120]; };
const ZitaTab& zita_tab () {                     // Resampler_table ctor, resampler-table.cc:29-44,52-75 (fr = 1, hl = 24, np = 4)
    static ZitaTab T; static bool done = false;
    if (!done) {
        const unsigned hl = 24, np = 4; const double fr = 1.0;
        for (unsigned j = 0; j <= np; ++j) {
            double t = (double)j / (double)np;
            for (unsigned i = 0; i < hl; ++i) {
                double x = fabs (t * fr), sc = 1.0;
                if (!(x < 1e-6)) { x *= M_PI; sc = sin (x) / x; }
                double y = fabs (t / hl), wd = 0.0;
                if (!(y >= 1.0)) { y *= M_PI; wd = 0.384 + 0.500 * cos (y) + 0.116 * cos (2 * y); }
                T.c[j * hl + hl - i - 1] = (float)(fr * sc * wd);
                t += 1;
            }
        }
        done = true;
    }
    return T;
}
// Steady state of Resampler::process (resampler.cc:171-262) after TruePeakdsp::init's 8192-zero pre-roll
// (truepeakdsp.cc:159-168: nread = 1, phase = 0): every input sample is appended to a 48-sample window and
// yields four outputs, phase ph using c1 = ctab + 24 ph (walking up from the oldest sample) and
// c2 = ctab + 24 (4 - ph) (walking down from the newest), pair-sum first, on a 1e-20f bias (:213-230).
struct Up4 {
    float w[48];                                 // w[0] oldest .. w[47] newest
    Up4 () { memset (w, 0, sizeof (w)); }
    inline void push (float x, float* out4) {
        memmove (w, w + 1, 47 * sizeof (float)); w[47] = x;
        const float* tab = zita_tab ().c;
        for (int ph = 0; ph < 4; ++ph) {
            const float* c1 = tab + 24 * ph; const float* c2 = tab + 24 * (4 - ph);
            float s = 1e-20f;
            for (int i = 0; i < 24; ++i) s += w[i] * c1[i] + w[47 - i] * c2[i];
            out4[ph] = s - 1e-20f;
        }
    }
};

// =====================================================================================
// True peak — jmeters/truepeakdsp.cc
// =====================================================================================
struct TruePeak {
    float m, p, z1, z2, w1, w2, w3, g; bool res; Up4 up;
    void init (float fs) {                       // :148-157
        z1 = z2 = .0f; m = p = 0; res = true;
        w1 = 4000.0f / fs / 4.0; w2 = 17200.0f / fs / 4.0; w3 = 1.0f - 7.0f / fs / 4.0; g = 0.502f;
    }
    void process (const float* d, int n) {       // :41-99
        float lm = res ? 0 : m, lp = res ? 0 : p;
        float a = z1 > 20 ? 20 : (z1 < 0 ? 0 : z1), b = z2 > 20 ? 20 : (z2 < 0 ? 0 : z2);
        float o[4];
        for (int k = 0; k < n; ++k) {
            up.push (d[k], o);
            a *= w3; b *= w3;
            for (int i = 0; i < 4; ++i) {
                float v = fabsf (o[i]);
                if (v > a) a += w1 * (v - a);
                if (v > b) b += w2 * (v - b);
                if (v > lp) lp = v;
            }
            float v = a + b;
            if (v > lm) lm = v;
        }
        z1 = a + 1e-20f; z2 = b + 1e-20f;
        lm *= g;
        if (res) { m = lm; p = lp; res = false; }
        else { if (lm > m) m = lm; if (lp > p) p = lp; }
    }
    void process_max (const float* d, int n) {   // :101-124
        float lm = res ? 0 : m, o[4];
        for (int k = 0; k < n; ++k) { up.push (d[k], o); for (int i = 0; i < 4; ++i) { float v = fabsf (o[i]); if (v > lm) lm = v; } }
        m = lm;
    }
};

// =====================================================================================
// K-meter — jmeters/kmeterdsp.cc
// =====================================================================================
struct Kmeter {
    float z1 = 0, z2 = 0, rms = 0, peak = 0, fall = 0; int cnt = 0, fpp = 0; bool flag = false;
    static float omega, fsamp; static int hold;
    static void init (float fs) { fsamp = fs; hold = (int)(0.5f * fs + 0.5f); omega = 9.72f / fs; }   // :47-54
    void process (const float* p, int n) {       // :56-140
        if (fpp != n) { fall = powf (10.0f, -0.05f * 15.0f * ((float)n / fsamp)); fpp = n; }
        float t = 0, a = z1 > 50 ? 50 : (z1 < 0 ? 0 : z1), b = z2 > 50 ? 50 : (z2 < 0 ? 0 : z2);
        for (int q = n / 4; q > 0; --q) {
            for (int i = 0; i < 4; ++i) { float s = *p++; s *= s; if (t < s) t = s; a += omega * (s - a); }
            b += 4 * omega * (a - b);
        }
        if (std::isnan (a)) a = 0;
        if (std::isnan (b)) b = 0;
        if (!fin (t)) t = 0;
        z1 = a + 1e-20f; z2 = b + 1e-20f;
        float s = sqrtf (2.0f * b); t = sqrtf (t);
        if (flag) { rms = s; flag = false; } else if (s > rms) rms = s;
        if (t >= peak) { peak = t; cnt = hold; }
        else if (cnt > 0) cnt -= fpp;
        else { peak *= fall; peak += 1e-10f; }
    }
    void reset () { z1 = z2 = rms = peak = .0f; cnt = 0; flag = false; }   // :157-162
};
float Kmeter::omega, Kmeter::fsamp; int Kmeter::hold;

// =====================================================================================
// Needle-meter ballistics — jmeters/vumeterdsp.cc, iec1ppmdsp.cc, iec2ppmdsp.cc, msppmdsp.cc
// =====================================================================================
struct Needle {                                  // one meter: kind 0 VU, 1 IEC-I, 2 IEC-II, 3 M/S PPM (mid), 4 M/S PPM (side)
    float z1 = 0, z2 = 0, m = 0; bool res = true; float db = 0, mv = 1.0f;
    static float w1, w2, w3, g;
    static void init (int kind, float fs) {
        if (kind == 0) { w1 = 11.1f / fs; w2 = w3 = 0; g = 1.5f * 1.571f; }                                  // vumeterdsp.cc:89-93
        else if (kind == 1) { w1 = 450.0f / fs; w2 = 1300.0f / fs; w3 = 1.0f - 5.4f / fs; g = 0.5108f; }     // iec1ppmdsp.cc:93-99
        else { w1 = 200.0f / fs; w2 = 860.0f / fs; w3 = 1.0f - 4.0f / fs; g = 0.5141f; }                     // iec2ppmdsp.cc:93-99, msppmdsp.cc:127-133
    }
    void set_gain (float d) { if (db == d) return; db = d; mv = powf (10, .05 * d); }                        // msppmdsp.cc:135-143
    void vu (const float* p, int n) {            // Vumeterdsp::process :45-73
        float a = z1 > 20 ? 20 : (z1 < -20 ? -20 : z1), b = z2 > 20 ? 20 : (z2 < -20 ? -20 : z2), mm = res ? 0 : m;
        res = false;
        for (int q = n / 4; q > 0; --q) {
            const float t2 = b / 2;
            for (int i = 0; i < 4; ++i) { const float t1 = fabsf (*p++) - t2; a += w1 * (t1 - a); }
            b += 4 * w1 * (a - b);
            if (b > mm) mm = b;
        }
        if (!fin (a)) { z1 = 0; mm = INFINITY; } else z1 = a;
        if (!fin (b)) { z2 = 0; mm = INFINITY; } else z2 = b + 1e-10f;
        m = mm;
    }
    // Iec1ppmdsp/Iec2ppmdsp::process (:47-80), Msppmdsp::processM/S (:50-118): t(i) yields the rectified sample
    template <class F> void ppm (int n, F t) {
        float a = z1 > 20 ? 20 : (z1 < 0 ? 0 : z1), b = z2 > 20 ? 20 : (z2 < 0 ? 0 : z2), mm = res ? 0 : m;
        res = false;
        int k = 0;
        for (int q = n / 4; q > 0; --q) {
            a *= w3; b *= w3;
            for (int i = 0; i < 4; ++i) { const float v = t (k++); if (v > a) a += w1 * (v - a); if (v > b) b += w2 * (v - b); }
            const float s = a + b;
            if (s > mm) mm = s;
        }
        z1 = a + 1e-10f; z2 = b + 1e-10f; m = mm;
    }
    float read () { res = true; return g * m; }
};
float Needle::w1, Needle::w2, Needle::w3, Needle::g;
struct NeedleBank { int n, kind; std::vector<Needle> v; };

// =====================================================================================
// Stereo correlation — jmeters/stcorrdsp.cc
// =====================================================================================
struct Stcorr {
    float zl = 0, zr = 0, zlr = 0, zll = 0, zrr = 0;
    static float w1, w2;
    static void init (int fs, float flp, float tcf) { w1 = 6.28f * flp / fs; w2 = 1 / (tcf * fs); }   // :85-93
    void process (const float* pl, const float* pr, int n) {   // :47-76
        float l = zl, r = zr, lr = zlr, ll = zll, rr = zrr;
        while (n--) {
            l += w1 * (*pl++ - l) + 1e-20f;
            r += w1 * (*pr++ - r) + 1e-20f;
            lr += w2 * (l * r - lr);
            ll += w2 * (l * l - ll);
            rr += w2 * (r * r - rr);
        }
        if (!fin (l)) l = 0; if (!fin (r)) r = 0; if (!fin (lr)) lr = 0; if (!fin (ll)) ll = 0; if (!fin (rr)) rr = 0;
        zl = l; zr = r; zlr = lr + 1e-10f; zll = ll + 1e-10f; zrr = rr + 1e-10f;
    }
    float read () const { return zlr / sqrtf (zll * zrr + 1e-10f); }   // :79-82
};
float Stcorr::w1, Stcorr::w2;

// =====================================================================================
// 30-band spectrum — src/spectr.c, src/spectrumlv2.c
// =====================================================================================
typedef std::complex<double> cd;
struct Biquad { double W[6]; double z[2]; };     // a0 a1 a2 b0 b1 b2 ; z1 z2   (spectr.c:54-60)
struct Band { Biquad f[6]; bool ac; };

// noinline/noclone: `order` must stay a run-time value.  If GCC specialises this routine for order = 6 it
// folds cos/sin of the (then constant) pole angles at compile time with MPFR, which differs from glibc's
// run-time cos/sin in the last ulp for some angles; the reference build (oracle/_ref) evaluates them at
// run time, and that is the behaviour pinned here.
__attribute__ ((noinline, noclone))
void band_design (Band& fb, double rate, double freq, double band, int order)   // bandpass_setup, spectr.c:89-206
{
    for (int i = 0; i < order; ++i) fb.f[i].z[0] = fb.f[i].z[1] = 0;
    fb.ac = false;
    const double wc = 2. * M_PI * freq / rate, ww = 2. * M_PI * band / rate;
    double wl = wc - (ww / 2.), wu = wc + (ww / 2.);
    if (wu > M_PI - 1e-9) wu = M_PI - 1e-9;
    if (wl < 1e-9) wl = 1e-9;
    wu *= .5; wl *= .5;
    const double c_a = cos (wu + wl) / cos (wu - wl);
    const double c_b = 1. / tan (wu - wl);
    const double w = 2. * atan (sqrt (tan (wu) * tan (wl)));
    const double c_a2 = c_a * c_a, c_b2 = c_b * c_b, ab_2 = 2. * c_a * c_b;
    const cd I (0.0, 1.0);
    for (int i = 0; i < order / 2; ++i) {
        const double om = M_PI_2 + (2 * i + 1) * M_PI / (2. * (double)order);
        cd p = cos (om) + I * sin (om);
        const cd c = (1. + p) / (1. - p);
        const cd d = 2 * (c_b - 1) * c + 2 * (1 + c_b);
        cd v = (4 * (c_b2 * (c_a2 - 1) + 1)) * c;
        v += 8 * (c_b2 * (c_a2 - 1) - 1);
        v *= c;
        v += 4 * (c_b2 * (c_a2 - 1) + 1);
        v = std::sqrt (v);
        const cd u0 = ab_2 + std::real (v * -1.) + ab_2 * std::real (c) + I * (std::imag (v * -1.) + ab_2 * std::imag (c));
        const cd u1 = ab_2 + std::real (v) + ab_2 * std::real (c) + I * (std::imag (v) + ab_2 * std::imag (c));
        const cd P0 = u0 / d, P1 = u1 / d;
        const cd Ps[2] = {P0, P1};
        for (int k = 0; k < 2; ++k) {
            double* W = fb.f[2 * i + k].W;
            W[0] = 1.; W[1] = -2 * std::real (Ps[k]);
            W[2] = std::real (Ps[k]) * std::real (Ps[k]) + std::imag (Ps[k]) * std::imag (Ps[k]);
            W[3] = 1.; W[4] = k ? -2. : 2.; W[5] = 1.;
        }
    }
    const double cos_w = cos (-w), sin_w = sin (-w), cos_w2 = cos (-2. * w), sin_w2 = sin (-2. * w);
    cd ch = 1, cb = 1;
    for (int i = 0; i < order; ++i) {
        const double* W = fb.f[i].W;
        ch *= ((1 + W[4] * cos_w) + cos_w2) + I * ((W[4] * sin_w) + sin_w2);
        cb *= ((1 + W[1] * cos_w) + W[2] * cos_w2) + I * ((W[1] * sin_w) + W[2] * sin_w2);
    }
    const cd scale = cb / ch;
    fb.f[0].W[3] *= std::real (scale); fb.f[0].W[4] *= std::real (scale); fb.f[0].W[5] *= std::real (scale);
}

inline float band_run (Band& fb, float in)       // bandpass_process + proc_one, spectr.c:68-87
{
    fb.ac = !fb.ac;
    double out = in + (fb.ac ? 1e-12 : -1e-12);
    for (int s = 0; s < 6; ++s) {
        Biquad& f = fb.f[s];
        const double y = f.W[3] * out + f.z[0];
        f.z[0] = f.W[4] * out - f.W[1] * y + f.z[1];
        f.z[1] = f.W[5] * out - f.W[2] * y;
        out = y;
    }
    return out;
}

struct Spec {
    int nchan; double rate; float rst_h, spd_h, omega, val[30], mx[30]; Band flt[30]; float ports[60];
    void init (int nc, double r) {               // spectrum_instantiate, spectrumlv2.c:73-121
        nchan = nc; rate = r; rst_h = -4; spd_h = 1.0;
        omega = 1.0f - expf (-2.0 * M_PI * spd_h / rate);
        const double f_r = 1000, b = 3, f1f = pow (2, -1. / (2. * b)), f2f = pow (2, 1. / (2. * b));
        for (int i = 0; i < 30; ++i) {
            const int x = i - 16;
            const double f_m = pow (2, x / b) * f_r, f_1 = f_m * f1f, f_2 = f_m * f2f;
            val[i] = mx[i] = 0;
            band_design (flt[i], rate, f_m, f_2 - f_1, 6);
        }
        memset (ports, 0, sizeof (ports));
    }
    void run (const float* l, const float* r, int n, float spd_p, float rst_p) {   // spectrum_run, :159-257
        bool reinit = false;
        if (spd_h != spd_p) {
            spd_h = spd_p; float v = spd_h;
            if (v < 0.01) v = 0.01;
            if (v > 15.0) v = 15.0;
            omega = 1.0f - expf (-2.0 * M_PI * v / rate);
            rst_h = 0;
        }
        if (rst_h != rst_p) {
            if (fabsf (rst_p) < 3 || rst_h == 0) { reinit = true; for (int i = 0; i < 30; ++i) mx[i] = 0; }
            if (fabsf (rst_p) != 3) rst_h = rst_p;
        }
        if (fabsf (rst_p) == 3) reinit = true;
        for (int j = 0; j < n; ++j) {
            const float in = nchan == 2 ? (l[j] + r[j]) / 2.0f : l[j];
            for (int i = 0; i < 30; ++i) {
                const float v = band_run (flt[i], in), s = v * v;
                val[i] += omega * (s - val[i]);
                if (val[i] > mx[i]) mx[i] = val[i];
            }
        }
        for (int i = 0; i < 30; ++i) {
            float vv = val[i];
            if (!fin (vv)) vv = 0;
            if (!fin (mx[i])) mx[i] = 0;
            for (int s = 0; s < 6; ++s) for (int q = 0; q < 2; ++q) if (!std::isfinite (flt[i].f[s].z[q])) flt[i].f[s].z[q] = 0;
            val[i] = vv + 1e-20f;
            const float vs = sqrtf (2. * vv), ms = sqrtf (2. * mx[i]);
            ports[i] = vs > .00001f ? 20.0 * log10f (vs) : -100.0;
            ports[30 + i] = reinit ? -500.0f : (ms > .00001f ? 20.0 * log10f (ms) : -100.0);   // reference: -500 - (rand() & 0xffff)
        }
    }
};

// =====================================================================================
// Bit-meter — src/bitmeter.c ; signal distribution histogram — src/sigdistlv2.c
// =====================================================================================
struct Bim {
    int32_t hist[584]; int zero, pos, nan_, inf_, den; float mn, mx; uint64_t itime; int resync; bool average, integrating; double rate;
    void clear () { memset (hist, 0, sizeof (hist)); mn = INFINITY; mx = 0; zero = pos = 0; itime = 0; }      // bim_clear :46-54
    void init (double r) { rate = r; average = false; integrating = true; resync = 0; clear (); nan_ = inf_ = den = 0; }   // :146-157, bim_reset :56-59
    void stats (const float* sp) {                      // float_stats :63-105
        uint32_t v; memcpy (&v, sp, 4);
        unsigned e = (v & 0x7f800000u) >> 23; const bool positive = !(v & 0x80000000u);
        v &= 0x7fffff;
        if (e == 255) { if (v == 0) ++inf_; else ++nan_; return; }
        if (e == 0 && v == 0) { ++zero; return; }
        if (e == 0) ++den;
        if (positive) ++pos;
        if (e > 0) {
            const float a = fabsf (*sp);
            if (a > mx) mx = a;
            if (a < mn) mn = a;
            ++hist[23 + e]; ++hist[303 + e];            // BIM_NHIT, BIM_NONE (src/uris.h:52-60)
        } else e = 1;
        for (int k = 0; k < 23; ++k) {
            ++hist[0 + e + k];                          // BIM_DHIT
            if (v & (1u << k)) { ++hist[280 + e + k]; ++hist[560 + k]; }   // BIM_DONE, BIM_DSET
        }
    }
    void run (const float* in, uint32_t n) {            // bim_run :248-327 (audio part + the ~5 fps window)
        if (integrating && itime < 2147483647) {
            if (itime > 2147483647 - n) itime = 2147483647;
            else { for (uint32_t s = 0; s < n; ++s) stats (in + s); itime += n; }
        }
        const int fps_limit = n * ceil (rate / (5.f * n));
        resync += n;
        if (resync >= fps_limit) { resync = resync % fps_limit; if (!average) clear (); }
    }
};
struct Sdh {
    int32_t hist[361]; int mx, peak; double avg, tmp, var; uint64_t itime; bool integrating;
    void init () { memset (hist, 0, sizeof (hist)); peak = -1; avg = tmp = var = 0; mx = 0; itime = 0; integrating = false; }   // sdh_instantiate :141-150
    void run (const float* in, uint32_t n) {            // sdh_run :287-327
        if (!(integrating && itime < 2147483647)) return;
        if (itime > 2147483647 - n) { itime = 2147483647; return; }
        for (uint32_t s = 0; s < n; ++s) {
            const float val = in[s];
            const float r = rintf (180.f + val * 150.f);
            if (!(r >= 0.f && r < 361.f)) continue;     // int conversion of NaN / out-of-range is INT_MIN on x86: "bin < 0"
            const int bin = (int)r;
            if ((++hist[bin]) > mx) { mx = hist[bin]; peak = bin; }
            avg += val;
            const double m1 = tmp, cnt = (double)(itime + s + 1);
            tmp = tmp + ((double)val - tmp) / cnt;
            var = var + ((double)val - tmp) * ((double)val - m1);
        }
        itime += n;
    }
};

// =====================================================================================
// Phasewheel FFT analysis — gui/fft.c, gui/phasewheel.c (FFTW replaced by a double-precision DFT)
// =====================================================================================
static void fft_pow2 (std::vector<std::complex<double>>& X)           // in place, iterative radix-2, double precision
{
    const int N = (int)X.size ();
    int lg = 0; while ((1 << lg) < N) ++lg;
    std::vector<std::complex<double>> T (N);
    for (int i = 0; i < N; ++i) { int r = 0; for (int b = 0; b < lg; ++b) if (i & (1 << b)) r |= 1 << (lg - 1 - b); T[r] = X[i]; }
    X.swap (T);
    for (int len = 2; len <= N; len <<= 1) {
        for (int i = 0; i < N; i += len)
            for (int k = 0; k < len / 2; ++k) {
                const double a = -2.0 * M_PI * k / len;
                const std::complex<double> w (cos (a), sin (a)), u = X[i + k], v = X[i + k + len / 2] * w;
                X[i + k] = u + v; X[i + k + len / 2] = u - v;
            }
    }
}
void dft_r2c (const float* in, int N, std::vector<std::complex<double>>& X)   // X_k = sum x_n e^{-2 pi i nk/N}
{
    // double precision: error ~1e-16, i.e. exact at float resolution.  N = 2^a, or 3 * 2^a (the GUI's 12288-point window,
    // gui/phasewheel.c:1115) by decimation in time: X_k = sum_r W_N^{rk} F_r[k mod N/3], F_r = DFT of x[3n + r]
    if (N % 3) { X.resize (N); for (int i = 0; i < N; ++i) X[i] = in[i]; fft_pow2 (X); return; }
    const int M = N / 3;
    std::vector<std::complex<double>> F[3];
    for (int r = 0; r < 3; ++r) { F[r].resize (M); for (int n = 0; n < M; ++n) F[r][n] = in[3 * n + r]; fft_pow2 (F[r]); }
    X.resize (N);
    for (int k = 0; k < N; ++k) {
        const double a1 = -2.0 * M_PI * k / N;
        X[k] = F[0][k % M] + std::complex<double> (cos (a1), sin (a1)) * F[1][k % M] + std::complex<double> (cos (2 * a1), sin (2 * a1)) * F[2][k % M];
    }
}
struct FftA {                                    // struct FFTAnalysis, gui/fft.c:43-64
    int N, bins; uint32_t rboff, smps, sps, step;
    std::vector<float> win, ring, fin_, power, phase;
    void init (int window, double rate, double fps) {    // fftx_init :208-237 + ft_gen_window (Hann) :69-79,122-161
        N = window; bins = window / 2; rboff = smps = step = 0; sps = (uint32_t)ceil (rate / fps);
        win.resize (N); ring.assign (N, 0.f); fin_.assign (N, 0.f); power.assign (bins, 0.f); phase.assign (bins, 0.f);
        double sum = 0.0; const double c = 2.0 * M_PI / (N - 1.0);
        for (int i = 0; i < N; ++i) { win[i] = .5 - .5 * cos (c * i); sum += win[i]; }
        const double isum = 2.0 / sum;
        for (int i = 0; i < N; ++i) win[i] *= isum;
    }
    int run1 (const float* d, uint32_t n) {      // _fftx_run :288-340
        const uint32_t off = rboff, old = N - n;
        for (uint32_t i = 0; i < n; ++i) { ring[(i + off) % N] = d[i]; fin_[old + i] = d[i]; }
        rboff = (rboff + n) % N;
        smps += n;
        if (smps < sps) return -1;
        step = smps; smps = 0;
        const uint32_t p0 = (off + n) % N;
        for (uint32_t i = 0; i < old; ++i) fin_[i] = ring[(p0 + i) % N];
        for (int i = 0; i < N; ++i) fin_[i] *= win[i];
        std::vector<std::complex<double>> X;
        dft_r2c (fin_.data (), N, X);
        power[0] = (float)X[0].real () * (float)X[0].real (); phase[0] = 0;     // ft_analyze :163-180
        for (int i = 1; i < bins - 1; ++i) {
            const float re = (float)X[i].real (), im = (float)X[i].imag ();
            power[i] = (re * re) + (im * im);
            phase[i] = atan2f (im, re);
        }
        return 0;
    }
    int run (const float* d, uint32_t n) {       // fftx_run :342-361
        if ((int)n <= N) return run1 (d, n);
        int rv = -1; uint32_t k = 0;
        while (k < n) { uint32_t s = (uint32_t)N < n - k ? N : n - k; if (!run1 (d + k, s)) rv = 0; k += s; }
        return rv;
    }
};
struct Pw {
    FftA a, b; int bins; std::vector<float> phase, level; float peak; int mode = 0;   // mode 1: stereoscope (phase[] holds lr[])
    void init (int fft_bins, double rate) {      // reinitialize_fft, gui/phasewheel.c:178-202
        bins = fft_bins; a.init (2 * bins, rate, 25); b.init (2 * bins, rate, 25);
        phase.assign (bins, 0.f); level.assign (bins, -100.f); peak = 0;
    }
    void set_mode (int m) {                      // stereoscope: reinitialize_fft, gui/stereoscope.c:143-146
        mode = m; phase.assign (bins, m ? 0.5f : 0.f); level.assign (bins, -100.f); peak = 0;
    }
    int process (const float* l, const float* r, int n, float thr) {   // process_audio :1307-1342
        a.run (l, n);
        const bool display = !b.run (r, n);
        if (display && mode == 1) {              // stereoscope process_audio, gui/stereoscope.c:705-741
            const float db_thresh = 1e-20;
            for (int i = 1; i < bins - 1; ++i) {
                if (a.power[i] < db_thresh && b.power[i] < db_thresh) { phase[i] = 0.5; level[i] = 0; continue; }
                const float lv = a.power[i] > b.power[i] ? a.power[i] : b.power[i];
                const float lr = .5 + .5 * (sqrtf (b.power[i]) - sqrtf (a.power[i])) / sqrtf (lv);
                level[i] += .1 * (lv - level[i]) + 1e-20;
                phase[i] += .1 * (lr - phase[i]) + 1e-10;
            }
            return 1;
        }
        if (display) {
            float pk = 0;
            for (int i = 1; i < bins - 1; ++i) {
                if (a.power[i] < thr || b.power[i] < thr) { phase[i] = 0; level[i] = -100; continue; }
                phase[i] = b.phase[i] - a.phase[i];
                level[i] = a.power[i] > b.power[i] ? a.power[i] : b.power[i];
                if (level[i] > pk) pk = level[i];
            }
            peak += .04 * (pk - peak) + 1e-15;
            if (std::isnan (peak)) peak = 0;
            if (peak > 1000) peak = 1000;
        }
        return display ? 1 : 0;
    }
};

// =====================================================================================
// DR-14 / TPnRMS — src/dr14.c
// =====================================================================================
struct Dr14 {
    static constexpr int BINS = 8000;            // DR_HISTBINS :45
    int nch; bool dr_mode; double rate; uint64_t n_sample_cnt, sample_count = 0, num_fragments = 0;
    TruePeak tp[2]; Kmeter km[2];
    float m_dbtp[2], m_peak[2], m_rms[2], rms_sum[2], peak_cur[2], peak_hist[2][2];
    std::vector<uint32_t> hist[2];
    float port[12];                              // v_rms[2] v_peak[2] m_peak[2] m_rms[2] dr[2] dr_total block_count

    static float coeff_to_db (float c) { if (c < .0001) return -80; return 20 * log10f (c); }       // :236-239
    static float db_to_coeff (float db) { if (db <= -80) return 0; return powf (10, 0.05 * db); }   // :241-244

    void init (int n_channels, double r, bool dr) {                                                  // dr14_instantiate :104-166
        nch = n_channels; dr_mode = dr; rate = r; n_sample_cnt = rintf (rate * 3.0);
        Kmeter::init (r);
        for (int c = 0; c < nch; ++c) { tp[c].init (r); km[c] = Kmeter (); m_rms[c] = m_peak[c] = -81; m_dbtp[c] = 0; rms_sum[c] = peak_cur[c] = 0;
                                        peak_hist[c][0] = peak_hist[c][1] = 0; if (dr) hist[c].assign (BINS, 0); }
        memset (port, 0, sizeof (port));
    }
    void reset_peaks () {                                                                            // :241-258
        for (int c = 0; c < nch; ++c) {
            m_peak[c] = -81; m_rms[c] = -81; m_dbtp[c] = 0; rms_sum[c] = 0; peak_cur[c] = 0; peak_hist[c][0] = peak_hist[c][1] = 0;
            km[c].reset ();
            if (dr_mode) std::fill (hist[c].begin (), hist[c].end (), 0u);
        }
        sample_count = 0; num_fragments = 0;
    }
    void calc_rms_score () {                                                                         // dr14_calc_rms_score :285-352
        bool silent = true;
        for (int c = 0; c < nch; ++c) if (rms_sum[c] > 1e-9 * (float)n_sample_cnt) silent = false;
        if (silent) { for (int c = 0; c < nch; ++c) rms_sum[c] = 0; return; }
        num_fragments++;
        const float mc = floorf (num_fragments / 5.0);
        const uint32_t m_cut = 1 > mc ? 1 : mc;
        for (int c = 0; c < nch; ++c) {
            const float rms = sqrt (2.f * rms_sum[c] / (float)n_sample_cnt);
            rms_sum[c] = 0;
            int bin = rintf (100.f * (80.f + coeff_to_db (rms))) - 1;
            if (bin >= BINS) bin = BINS - 1;
            if (bin > 0) hist[c][bin]++;
            uint32_t n_cut = 0; float rms_score = 0;
            if (num_fragments > 2)
                for (int32_t b = BINS - 1; b > 0 && n_cut < m_cut; --b) {
                    const uint32_t bc = hist[c][b];
                    if (bc == 0) continue;
                    const float cd = db_to_coeff ((b - BINS + 1) / 100.0);
                    rms_score += cd * cd * (float)bc;
                    n_cut += bc;
                }
            m_rms[c] = n_cut > 0 ? coeff_to_db (sqrtf (rms_score / n_cut)) : -81;
            if (peak_cur[c] >= peak_hist[c][0]) { peak_hist[c][1] = peak_hist[c][0]; peak_hist[c][0] = peak_cur[c]; }
            else if (peak_cur[c] > peak_hist[c][1]) peak_hist[c][1] = peak_cur[c];
            peak_cur[c] = 0;
            m_peak[c] = num_fragments > 2 ? coeff_to_db (peak_hist[c][1]) : -81;
        }
    }
    void run (const float* const* in, int n) {                                                        // dr14_run :391-462 (no atoms, button up)
        for (int c = 0; c < nch; ++c) { km[c].process (in[c], n); tp[c].process (in[c], n); }
        if (dr_mode) {
            uint64_t scnt = sample_count;
            for (int s = 0; s < n; ++s) {
                for (int c = 0; c < nch; ++c) { const float v = in[c][s]; rms_sum[c] += v * v; peak_cur[c] = peak_cur[c] > v ? peak_cur[c] : v; }
                if (++scnt > n_sample_cnt) { calc_rms_score (); scnt = 0; }
            }
            sample_count = scnt;
        }
        float dr_total = 0; int dr_valid = 0;
        for (int c = 0; c < nch; ++c) {
            const float pv = tp[c].m, pp = tp[c].p; tp[c].res = true;                               // read (pv, pp)
            const float rv = km[c].rms, rp = km[c].peak; km[c].flag = true;                         // read (rv, rp)
            m_dbtp[c] = m_dbtp[c] > pp ? m_dbtp[c] : pp;
            port[0 + c] = coeff_to_db (rv); port[2 + c] = coeff_to_db (pv); port[4 + c] = coeff_to_db (m_dbtp[c]);
            if (dr_mode) {
                const float rdb = m_rms[c], pdb = m_peak[c];
                const float dr = (0 < pdb ? 0 : pdb) - rdb;
                if (rdb > -80 && pdb > -80) { dr_total += dr; dr_valid++; }
                const float lo = 20 < dr ? 20 : dr;
                port[8 + c] = (rdb > -80 && pdb > -80) ? (1 > lo ? 1 : lo) : 21;
                port[6 + c] = rdb;
            } else port[6 + c] = coeff_to_db (rp);
        }
        if (nch > 1 && dr_mode) {
            if (dr_valid > 0) { const float a = dr_total / (float)dr_valid; const float lo = 20 < a ? 20 : a; port[10] = 1 > lo ? 1 : lo; }
            else port[10] = 21;
        }
        port[11] = 3.0 * num_fragments;
    }
};

template <class T> struct Bank { int n, nchan; std::vector<T> v; };

}  // namespace

// =====================================================================================
// extern "C" API (oracle_api.h)
// =====================================================================================
extern "C" {

const char* orc_kind (void) { return "port"; }
int orc_hw_threads (void) { return (int)std::thread::hardware_concurrency (); }

void* orc_ebu_create (int n, int nchan, float fs) { auto* b = new Bank<Ebu>; b->n = n; b->nchan = nchan; b->v.resize (n); for (auto& e : b->v) e.init (nchan, fs); return b; }
void orc_ebu_destroy (void* h) { delete (Bank<Ebu>*)h; }
void orc_ebu_integr (void* h, int inst, int cmd) {
    auto* b = (Bank<Ebu>*)h;
    for (int i = 0; i < b->n; ++i) { if (inst >= 0 && i != inst) continue; if (cmd == 0) b->v[i].integr = false; else if (cmd == 1) b->v[i].integr = true; else b->v[i].integr_reset (); }
}
void orc_ebu_reset (void* h, int inst) { auto* b = (Bank<Ebu>*)h; for (int i = 0; i < b->n; ++i) if (inst < 0 || i == inst) b->v[i].reset (); }
void orc_ebu_process (void* h, const float* in, size_t stride, int nfram, int nthreads) {
    auto* b = (Bank<Ebu>*)h;
    par_for (b->n, nthreads, [=] (int a, int e) {
        for (int i = a; i < e; ++i) { const float* ip[5]; for (int c = 0; c < b->nchan; ++c) ip[c] = in + ((size_t)i * b->nchan + c) * stride; b->v[i].process (nfram, ip); }
    });
}
void orc_ebu_read (void* h, float* out) {
    auto* b = (Bank<Ebu>*)h;
    for (int i = 0; i < b->n; ++i) { const Ebu& e = b->v[i]; float* o = out + 9 * i; o[0] = e.lM; o[1] = e.mM; o[2] = e.lS; o[3] = e.mS; o[4] = e.integ; o[5] = e.ithr; o[6] = e.rmin; o[7] = e.rmax; o[8] = e.rthr; }
}
void orc_ebu_hist (void* h, int inst, int* hm, int* hs, int* c4) {
    const Ebu& e = ((Bank<Ebu>*)h)->v[inst];
    memcpy (hm, e.hM.bins, sizeof (e.hM.bins)); memcpy (hs, e.hS.bins, sizeof (e.hS.bins));
    c4[0] = e.hM.count; c4[1] = e.hS.count; c4[2] = e.hM.error; c4[3] = e.hS.error;
}
void orc_ebu_hist_calc (const int* hm, int cm, const int* hs, int cs, float* o) {   // calc_integ + calc_range (:105-150) on given counts
    Hist M, S;
    memcpy (M.bins, hm, sizeof (M.bins)); M.count = cm; M.error = 0;
    memcpy (S.bins, hs, sizeof (S.bins)); S.count = cs; S.error = 0;
    binpow_init ();
    for (int q = 0; q < 5; ++q) o[q] = -200.0f;
    hist_integ (M, o + 0, o + 1);
    hist_range (S, o + 2, o + 3, o + 4);
}
void orc_ebu_coeffs (void* h, float* o) { const Ebu& e = ((Bank<Ebu>*)h)->v[0]; o[0] = e.a0; o[1] = e.a1; o[2] = e.a2; o[3] = e.b1; o[4] = e.b2; o[5] = e.c3; o[6] = e.c4; }
void orc_ebu_state (void* h, int inst, float* z, float* pw, float* frpwr, int* c4) {
    auto* b = (Bank<Ebu>*)h; const Ebu& e = b->v[inst];
    for (int c = 0; c < b->nchan; ++c) for (int q = 0; q < 4; ++q) z[4 * c + q] = e.z[c][q];
    memcpy (pw, e.power, sizeof (e.power)); *frpwr = e.frpwr;
    c4[0] = e.frcnt; c4[1] = e.wrind; c4[2] = e.div1; c4[3] = e.div2;
}

void* orc_tp_create (int n, float fs) { auto* b = new Bank<TruePeak>; b->n = n; b->v.resize (n); for (auto& t : b->v) t.init (fs); return b; }
void orc_tp_destroy (void* h) { delete (Bank<TruePeak>*)h; }
void orc_tp_process (void* h, const float* in, size_t stride, int nfram, int mode, int nthreads) {
    auto* b = (Bank<TruePeak>*)h;
    par_for (b->n, nthreads, [=] (int a, int e) { for (int i = a; i < e; ++i) { if (mode) b->v[i].process_max (in + (size_t)i * stride, nfram); else b->v[i].process (in + (size_t)i * stride, nfram); } });
}
void orc_tp_read (void* h, float* m, float* p) { auto* b = (Bank<TruePeak>*)h; for (int i = 0; i < b->n; ++i) { b->v[i].res = true; m[i] = b->v[i].m; p[i] = b->v[i].p; } }   // read(m,p) :133-138
void orc_tp_peek (void* h, float* m, float* p, float* z1, float* z2, int* res) {
    auto* b = (Bank<TruePeak>*)h;
    for (int i = 0; i < b->n; ++i) { const TruePeak& t = b->v[i]; m[i] = t.m; p[i] = t.p; z1[i] = t.z1; z2[i] = t.z2; res[i] = t.res; }
}
void orc_tp_reset (void* h, int inst) { auto* b = (Bank<TruePeak>*)h; for (int i = 0; i < b->n; ++i) if (inst < 0 || i == inst) { b->v[i].res = true; b->v[i].m = 0; b->v[i].p = 0; } }   // :140-145
void orc_tp_coeffs (void* h, float* w4, float* ctab) { const TruePeak& t = ((Bank<TruePeak>*)h)->v[0]; w4[0] = t.w1; w4[1] = t.w2; w4[2] = t.w3; w4[3] = t.g; memcpy (ctab, zita_tab ().c, 120 * sizeof (float)); }
void orc_tp_upsample (float, const float* in, int n, int, float* out) { Up4 u; for (int k = 0; k < n; ++k) u.push (in[k], out + 4 * k); }

void orc_r128_cycle (void* eh, void* th, const float* in, size_t stride, int nfram, int nblocks, int nthreads) {
    auto* e = (Bank<Ebu>*)eh; auto* t = (Bank<TruePeak>*)th;
    par_for (e->n, nthreads, [=] (int a, int b) {
        for (int i = a; i < b; ++i)
            for (int blk = 0; blk < nblocks; ++blk) {
                const float* l = in + (size_t)(2 * i) * stride + (size_t)blk * nfram;
                const float* r = in + (size_t)(2 * i + 1) * stride + (size_t)blk * nfram;
                const float* ip[2] = {l, r};
                e->v[i].process (nfram, ip);
                if (t) { t->v[2 * i].process_max (l, nfram); t->v[2 * i + 1].process_max (r, nfram); t->v[2 * i].res = true; t->v[2 * i + 1].res = true; }
            }
    });
}

void* orc_km_create (int n, float fs) { auto* b = new Bank<Kmeter>; b->n = n; b->v.resize (n); Kmeter::init (fs); return b; }
void orc_km_destroy (void* h) { delete (Bank<Kmeter>*)h; }
void orc_km_process (void* h, const float* in, size_t stride, int nfram, int nthreads) {
    auto* b = (Bank<Kmeter>*)h;
    par_for (b->n, nthreads, [=] (int a, int e) { for (int i = a; i < e; ++i) b->v[i].process (in + (size_t)i * stride, nfram); });
}
void orc_km_read (void* h, float* rms, float* peak) { auto* b = (Bank<Kmeter>*)h; for (int i = 0; i < b->n; ++i) { rms[i] = b->v[i].rms; peak[i] = b->v[i].peak; b->v[i].flag = true; } }   // :150-155
void orc_km_peek (void* h, float* s) {
    auto* b = (Bank<Kmeter>*)h;
    for (int i = 0; i < b->n; ++i) { const Kmeter& k = b->v[i]; float* o = s + 8 * i; o[0] = k.z1; o[1] = k.z2; o[2] = k.rms; o[3] = k.peak; o[4] = k.fall; o[5] = (float)k.cnt; o[6] = (float)k.fpp; o[7] = k.flag; }
}
void orc_km_reset (void* h, int inst) { auto* b = (Bank<Kmeter>*)h; for (int i = 0; i < b->n; ++i) if (inst < 0 || i == inst) b->v[i].reset (); }
void orc_km_coeffs (void*, float* omega, int* hold) { *omega = Kmeter::omega; *hold = Kmeter::hold; }

void* orc_ppm_create (int n, float fs, int kind) {
    auto* b = new NeedleBank; b->n = n; b->kind = kind; b->v.resize (kind == 3 ? 2 * n : n); Needle::init (kind, fs);
    if (kind == 3) for (auto& m : b->v) m.set_gain (-6);
    return b;
}
void orc_ppm_destroy (void* h) { delete (NeedleBank*)h; }
void orc_ppm_process (void* h, const float* in, size_t stride, int nfram, int nthreads) {
    auto* b = (NeedleBank*)h;
    par_for (b->n, nthreads, [=] (int a, int e) {
        for (int i = a; i < e; ++i) {
            if (b->kind == 0) b->v[i].vu (in + (size_t)i * stride, nfram);
            else if (b->kind < 3) { const float* p = in + (size_t)i * stride; b->v[i].ppm (nfram, [=] (int k) { return fabsf (p[k]); }); }
            else {
                const float* l = in + (size_t)(2 * i) * stride; const float* r = l + stride;
                Needle& M = b->v[2 * i]; Needle& S = b->v[2 * i + 1];
                const float gm = M.mv, gs = S.mv;
                M.ppm (nfram, [=] (int k) { return gm * fabsf (l[k] + r[k]); });
                S.ppm (nfram, [=] (int k) { return gs * fabsf (l[k] - r[k]); });
            }
        }
    });
}
void orc_ppm_read (void* h, float* out) { auto* b = (NeedleBank*)h; for (size_t i = 0; i < b->v.size (); ++i) out[i] = b->v[i].read (); }
void orc_ppm_peek (void* h, float* s) { auto* b = (NeedleBank*)h; for (size_t i = 0; i < b->v.size (); ++i) { s[4 * i] = b->v[i].z1; s[4 * i + 1] = b->v[i].z2; s[4 * i + 2] = b->v[i].m; s[4 * i + 3] = b->v[i].res; } }
void orc_ppm_set_gain (void* h, float db_m, float db_s) { auto* b = (NeedleBank*)h; if (b->kind != 3) return; for (int i = 0; i < b->n; ++i) { b->v[2 * i].set_gain (db_m); b->v[2 * i + 1].set_gain (db_s); } }
void orc_ppm_coeffs (void* h, float* w) { (void)h; w[0] = Needle::w1; w[1] = Needle::w2; w[2] = Needle::w3; w[3] = Needle::g; }

void* orc_cor_create (int n, int fs, float flp, float tcf) { auto* b = new Bank<Stcorr>; b->n = n; b->v.resize (n); Stcorr::init (fs, flp, tcf); return b; }
void orc_cor_destroy (void* h) { delete (Bank<Stcorr>*)h; }
void orc_cor_process (void* h, const float* in, size_t stride, int nfram, int nthreads) {
    auto* b = (Bank<Stcorr>*)h;
    par_for (b->n, nthreads, [=] (int a, int e) { for (int i = a; i < e; ++i) b->v[i].process (in + (size_t)(2 * i) * stride, in + (size_t)(2 * i + 1) * stride, nfram); });
}
void orc_cor_read (void* h, float* out) { auto* b = (Bank<Stcorr>*)h; for (int i = 0; i < b->n; ++i) out[i] = b->v[i].read (); }
void orc_cor_peek (void* h, float* s) { auto* b = (Bank<Stcorr>*)h; for (int i = 0; i < b->n; ++i) { const Stcorr& c = b->v[i]; float* o = s + 5 * i; o[0] = c.zl; o[1] = c.zr; o[2] = c.zlr; o[3] = c.zll; o[4] = c.zrr; } }
void orc_cor_coeffs (void*, float* w) { w[0] = Stcorr::w1; w[1] = Stcorr::w2; }

void* orc_spec_create (int n, int nchan, double rate) { auto* b = new Bank<Spec>; b->n = n; b->nchan = nchan; b->v.resize (n); for (auto& s : b->v) s.init (nchan, rate); return b; }
void orc_spec_destroy (void* h) { delete (Bank<Spec>*)h; }
void orc_spec_process (void* h, const float* in, size_t stride, int nfram, float speed, float reset, int nthreads) {
    auto* b = (Bank<Spec>*)h;
    par_for (b->n, nthreads, [=] (int a, int e) {
        for (int i = a; i < e; ++i) { const float* l = in + (size_t)i * b->nchan * stride; b->v[i].run (l, b->nchan == 2 ? l + stride : l, nfram, speed, reset); }
    });
}
void orc_spec_read (void* h, float* out) { auto* b = (Bank<Spec>*)h; for (int i = 0; i < b->n; ++i) memcpy (out + 60 * i, b->v[i].ports, 60 * sizeof (float)); }
void orc_spec_state (void* h, int inst, double* z, float* v, float* m) {
    const Spec& s = ((Bank<Spec>*)h)->v[inst];
    for (int b = 0; b < 30; ++b) { v[b] = s.val[b]; m[b] = s.mx[b]; for (int q = 0; q < 6; ++q) { z[(b * 6 + q) * 2] = s.flt[b].f[q].z[0]; z[(b * 6 + q) * 2 + 1] = s.flt[b].f[q].z[1]; } }
}
void orc_spec_coeffs (void* h, double* W) { const Spec& s = ((Bank<Spec>*)h)->v[0]; for (int b = 0; b < 30; ++b) for (int q = 0; q < 6; ++q) for (int k = 0; k < 6; ++k) W[(b * 6 + q) * 6 + k] = s.flt[b].f[q].W[k]; }

void* orc_ebuplug_create (int, float, int) { return 0; }       // the plugin glue itself exists only as the reference build
void  orc_ebuplug_destroy (void*) {}
void  orc_ebuplug_run (void*, const float*, size_t, int, int) {}
void  orc_ebuplug_read (void*, float*) {}
void* orc_bim_create (int n, float rate) { auto* b = new Bank<Bim>; b->n = n; b->v.resize (n); for (auto& m : b->v) m.init (rate); return b; }
void  orc_bim_destroy (void* h) { delete (Bank<Bim>*)h; }
void  orc_bim_mode (void* h, int average, int integrating) { for (auto& m : ((Bank<Bim>*)h)->v) { m.average = average; m.integrating = integrating; } }
void  orc_bim_process (void* h, const float* in, size_t stride, int nfram, int nthreads) {
    auto* b = (Bank<Bim>*)h;
    par_for (b->n, nthreads, [=] (int a, int e) { for (int i = a; i < e; ++i) b->v[i].run (in + (size_t)i * stride, (uint32_t)nfram); });
}
void  orc_bim_read (void* h, int inst, int32_t* hist, int32_t* c, float* mm, int64_t* it) {
    const Bim& m = ((Bank<Bim>*)h)->v[inst];
    memcpy (hist, m.hist, sizeof (m.hist)); c[0] = m.zero; c[1] = m.pos; c[2] = m.nan_; c[3] = m.inf_; c[4] = m.den; mm[0] = m.mn; mm[1] = m.mx; *it = (int64_t)m.itime;
}
void* orc_sdh_create (int n, float) { auto* b = new Bank<Sdh>; b->n = n; b->v.resize (n); for (auto& m : b->v) m.init (); return b; }
void  orc_sdh_destroy (void* h) { delete (Bank<Sdh>*)h; }
void  orc_sdh_integrate (void* h, int on) { for (auto& m : ((Bank<Sdh>*)h)->v) m.integrating = on; }
void  orc_sdh_process (void* h, const float* in, size_t stride, int nfram, int nthreads) {
    auto* b = (Bank<Sdh>*)h;
    par_for (b->n, nthreads, [=] (int a, int e) { for (int i = a; i < e; ++i) b->v[i].run (in + (size_t)i * stride, (uint32_t)nfram); });
}
void  orc_sdh_read (void* h, int inst, int32_t* hist, int32_t* mp, double* av, int64_t* it) {
    const Sdh& m = ((Bank<Sdh>*)h)->v[inst];
    memcpy (hist, m.hist, sizeof (m.hist)); mp[0] = m.mx; mp[1] = m.peak; av[0] = m.avg; av[1] = m.tmp; av[2] = m.var; *it = (int64_t)m.itime;
}

void* orc_dr14_create (int n, int nch, double rate, int dr_mode) { auto* b = new Bank<Dr14>; b->n = n; b->nchan = nch; b->v.resize (n); for (auto& d : b->v) d.init (nch, rate, dr_mode != 0); return b; }
void orc_dr14_destroy (void* h) { delete (Bank<Dr14>*)h; }
void orc_dr14_process (void* h, const float* in, size_t stride, int nfram, int nthreads) {
    auto* b = (Bank<Dr14>*)h;
    par_for (b->n, nthreads, [=] (int a, int e) { for (int i = a; i < e; ++i) { const float* ip[2] = {in + (size_t)(i * b->nchan) * stride, in + (size_t)(i * b->nchan + b->nchan - 1) * stride}; b->v[i].run (ip, nfram); } });
}
void orc_dr14_reset (void* h) { for (auto& d : ((Bank<Dr14>*)h)->v) d.reset_peaks (); }
void orc_dr14_read (void* h, float* out) { auto* b = (Bank<Dr14>*)h; for (int i = 0; i < b->n; ++i) memcpy (out + 12 * i, b->v[i].port, sizeof (b->v[i].port)); }

void* orc_pw_create (int n, int fft_bins, double rate) { auto* b = new Bank<Pw>; b->n = n; b->v.resize (n); for (auto& p : b->v) p.init (fft_bins, rate); return b; }
void orc_pw_destroy (void* h) { delete (Bank<Pw>*)h; }
void orc_pw_set_mode (void* h, int mode) { for (auto& p : ((Bank<Pw>*)h)->v) p.set_mode (mode); }
int orc_pw_process (void* h, const float* in, size_t stride, int nfram, float thr, int nthreads) {
    auto* b = (Bank<Pw>*)h; std::vector<int> fired (b->n, 0);
    par_for (b->n, nthreads, [&] (int a, int e) { for (int i = a; i < e; ++i) fired[i] = b->v[i].process (in + (size_t)(2 * i) * stride, in + (size_t)(2 * i + 1) * stride, nfram, thr); });
    return fired[0];
}
void orc_pw_read (void* h, float* phase, float* level, float* peak) {
    auto* b = (Bank<Pw>*)h;
    for (int i = 0; i < b->n; ++i) { const Pw& p = b->v[i]; memcpy (phase + (size_t)i * p.bins, p.phase.data (), p.bins * 4); memcpy (level + (size_t)i * p.bins, p.level.data (), p.bins * 4); peak[i] = p.peak; }
}
void orc_pw_raw (void* h, int inst, float* pl, float* pr, float* fl, float* fr) {
    const Pw& p = ((Bank<Pw>*)h)->v[inst];
    memcpy (pl, p.a.power.data (), p.bins * 4); memcpy (pr, p.b.power.data (), p.bins * 4);
    memcpy (fl, p.a.phase.data (), p.bins * 4); memcpy (fr, p.b.phase.data (), p.bins * 4);
}

}  // extern "C"

#include "cpu_bench.inc"
