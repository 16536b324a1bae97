// _ebu_weighted.cc — CPU restatement of Ebu_r128_proc (ebumeter/ebu_r128_proc.{h,cc} of x42/meters.lv2) for instances of 1..32
// channels with caller-given channel weights: the oracle of the weighted EBU R128 banks (b200m_ebu_create_weighted).
//
// TEST INFRASTRUCTURE ONLY: compiled by tests/_ebu_weighted.py into a temporary directory with the reference's float flags
// (SSE2 arithmetic, no FMA contraction) and loaded by the tests; the product never links it.  The per-chunk channel sum is
// detect_process's  si = 0; si += gain[i] * sj  (:324-330) for every channel, mono included, so with the reference's own weights
// (mono {2}, else 1 1 1 1.41 1.41) it is Ebu_r128_proc itself: tests/test_r128_weighted_cpu.py pins that bit for bit against the
// reference build.
#include <math.h>
#include <stddef.h>
#include <string.h>
#include <cmath>
#include <vector>

namespace {

constexpr int MAXCH = 32;
inline bool fin (float v) { return std::isfinite (v); }

float g_binpow[100];                            // _bin_power, initstat :54-63
void binpow_init () { if (g_binpow[0]) return; for (int i = 0; i < 100; ++i) g_binpow[i] = powf (10.0f, i / 100.0f); }

struct Hist {                                   // Ebu_r128_hist, :32-150
    int bins[751]; int count, error;
    void clear () { memset (bins, 0, sizeof (bins)); count = error = 0; }
    void add (float v) {                        // addpoint :66-79
        int k = (int)floorf (10 * v + 700.5f);
        if (k < 0) return;
        if (k > 750) { k = 750; error++; }
        bins[k]++; count++;
    }
    float mean (int i) const {                  // integrate :82-102
        int j = i % 100, n = 0; float s = 0;
        while (i <= 750) {
            int k = bins[i++];
            n += k;
            s += k * g_binpow[j++];
            if (j == 100) { j = 0; s /= 10.0f; }
        }
        return s / n;
    }
    void integ (float* vi, float* th) const {   // calc_integ :105-125
        if (count < 50) { *vi = -200.0f; return; }
        float s = mean (0);
        *th = 10 * log10f (s) - 10.0f;
        int k = (int)(floorf (100 * log10f (s) + 0.5f)) + 600;
        if (k < 0) k = 0;
        s = mean (k);
        *vi = 10 * log10f (s);
    }
    void range (float* v0, float* v1, float* th) const {   // calc_range :128-150
        if (count < 20) { *v0 = -200.0f; *v1 = -200.0f; return; }
        float s = mean (0);
        *th = 10 * log10f (s) - 20.0f;
        int k = (int)(floorf (100 * log10f (s) + 0.5)) + 500;   // 0.5 is a double literal in the reference
        if (k < 0) k = 0;
        int i, j, n;
        for (i = k, n = 0; i <= 750; i++) n += bins[i];
        const float a = 0.10f * n, b = 0.95f * n;
        for (i = k, s = 0; s < a; i++) s += bins[i];
        for (j = 750, s = n; s > b; j--) s -= bins[j];
        *v0 = (i - 701) / 10.0f;
        *v1 = (j - 699) / 10.0f;
    }
};

struct Ebu {
    int nchan, fragm, frcnt, wrind, div1, div2; bool integr;
    float frpwr, power[64], gain[MAXCH];
    float lM, mM, lS, mS, integ, ithr, rmin, rmax, rthr;
    float a0, a1, a2, b1, b2, c3, c4;
    float z[MAXCH][4];
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
    void init (int nc, float fs, const float* g) {
        nchan = nc; fragm = (int)fs / 20; design (fs); binpow_init ();
        for (int c = 0; c < nc; ++c) gain[c] = g[c];
        reset ();
    }
    float detect (const float* const* ip, int n) {          // detect_process :302-337 with the caller's weights
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
            si += gain[c] * sj;
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
        const float* ip[MAXCH];
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
                    if (++div2 == 10) { hS.add (lS); div2 = 0; hM.integ (&integ, &ithr); hS.range (&rmin, &rmax, &rthr); }
                }
            }
            for (int c = 0; c < nchan; ++c) ip[c] += k;
            nfram -= k;
        }
    }
};

struct Bank { int n, nchan; std::vector<Ebu> v; };

}  // namespace

extern "C" {

// n instances of nchan = 1..32 channels with weights gains[0..nchan); NULL outside 1..32.  Rows of a process call: inst * nchan + c.
void* ew_create (int n, int nchan, const float* gains, float fs)
{
    if (nchan < 1 || nchan > MAXCH || n < 1) return nullptr;
    Bank* b = new Bank; b->n = n; b->nchan = nchan; b->v.resize (n);
    for (auto& e : b->v) e.init (nchan, fs, gains);
    return b;
}
void ew_destroy (void* h) { delete (Bank*)h; }
void ew_integr (void* h, int inst, int cmd)     // 0 pause 1 start 2 reset (integr_reset); inst < 0: all
{
    Bank* b = (Bank*)h;
    for (int i = 0; i < b->n; ++i) {
        if (inst >= 0 && i != inst) continue;
        Ebu& e = b->v[i];
        if (cmd == 0) e.integr = false; else if (cmd == 1) e.integr = true; else e.integr_reset ();
    }
}
void ew_reset (void* h, int inst) { Bank* b = (Bank*)h; for (int i = 0; i < b->n; ++i) if (inst < 0 || i == inst) b->v[i].reset (); }
void ew_process (void* h, const float* in, size_t stride, int nfram)
{
    Bank* b = (Bank*)h;
    for (int i = 0; i < b->n; ++i) {
        const float* ip[MAXCH];
        for (int c = 0; c < b->nchan; ++c) ip[c] = in + ((size_t)i * b->nchan + c) * stride;
        b->v[i].process (nfram, ip);
    }
}
void ew_read (void* h, float* out)              // [n][9]: M maxM S maxS I Ithr Rmin Rmax Rthr
{
    Bank* b = (Bank*)h;
    for (int i = 0; i < b->n; ++i) {
        const Ebu& e = b->v[i]; float* o = out + 9 * i;
        o[0] = e.lM; o[1] = e.mM; o[2] = e.lS; o[3] = e.mS; o[4] = e.integ; o[5] = e.ithr; o[6] = e.rmin; o[7] = e.rmax; o[8] = e.rthr;
    }
}
void ew_hist (void* h, int inst, int* hm, int* hs, int* c4)   // 751, 751, {count M, count S, error M, error S}
{
    const Ebu& e = ((Bank*)h)->v[inst];
    memcpy (hm, e.hM.bins, sizeof (e.hM.bins)); memcpy (hs, e.hS.bins, sizeof (e.hS.bins));
    c4[0] = e.hM.count; c4[1] = e.hS.count; c4[2] = e.hM.error; c4[3] = e.hS.error;
}

}  // extern "C"
