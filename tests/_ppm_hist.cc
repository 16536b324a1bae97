// _ppm_hist.cc — the distribution of the needle meters' per-group readings: the oracle of the needle-meter bank's histogram plane
// (b200m_ppm_hist_enable / b200m_ppm_hist_read).
//
// TEST INFRASTRUCTURE ONLY: compiled by tests/_ppm_hist.py into a temporary directory with the reference's float flags (SSE2
// arithmetic, no FMA contraction) and loaded by the tests; the product never links it.
//
// ph_run continues every meter's process() (jmeters/vumeterdsp.cc:45-73, iec1ppmdsp.cc / iec2ppmdsp.cc:47-80,
// msppmdsp.cc:50-118) from a copy of its z1 z2 m res, taken from an oracle needle bank (_oracle.Needle.peek) just before the oracle
// runs the same block: the clamp at call start, "n /= 4" groups, the M/S gains, and the end-of-call scrub and bias.  After each
// group it takes the needle value s the reference compares with m (VU: z2; the others: t = z1 + z2), forms v = g * s and applies
// the rules of include/b200meters.h: the bin #{k : v >= e[k]} counted by a plain scan of the edge table, nonfinite, peak and the over
// runs against lim.  tests/_ppm_hist.py then checks the copies' end state bit for bit against the oracle's after its run.
#include <math.h>
#include <stddef.h>
#include <stdint.h>

struct Stats { uint64_t nonfinite, over_groups, overs, longest_over, run; float peak; uint32_t pad; };

static void tally (float g, float lim, const float* e, float s, uint64_t* c, Stats* a)
{
    const float v = g * s;
    if (!isfinite (v)) { a->nonfinite += 1; return; }
    if (v > a->peak) a->peak = v;
    if (v >= lim) {
        a->over_groups += 1;
        if (a->run == 0) a->overs += 1;
        a->run += 1;
        if (a->run > a->longest_over) a->longest_over = a->run;
    } else a->run = 0;
    int k = 0;
    while (k < 241 && v >= e[k]) ++k;
    c[k] += 1;
}

// kind 0 VU, 1 / 2 IEC I / II, 3 M/S (n pairs, rows 2i / 2i + 1, meters 2i = M, 2i + 1 = S); w = w1 w2 w3 g (b200m_design_ppm)
extern "C" void ph_run (int n, int kind, const float* w, float lim, float db_m, float db_s, float* state /* [nm][4] z1 z2 m res */,
                        const float* in, size_t stride, int nfram, const float* edges /* [241] */, uint64_t* counts /* [nm][242] */,
                        Stats* stats /* [nm] */)
{
    const float w1 = w[0], w2 = w[1], w3 = w[2], g = w[3];
    const int per = kind == 3 ? 2 : 1;
    float mvv[2] = {1.0f, 1.0f};                               // Msppmdsp (-6) then set_gain: _mv = powf (10, .05 * db) (msppmdsp.cc:135-143)
    if (db_m != 0) mvv[0] = powf (10, .05 * db_m);
    if (db_s != 0) mvv[1] = powf (10, .05 * db_s);
    for (int i = 0; i < n; ++i) {
        for (int q = 0; q < per; ++q) {
            const int mi = per * i + q;
            float* st = state + 4 * mi;
            uint64_t* c = counts + (size_t)mi * 242;
            Stats* a = stats + mi;
            float z1, z2, m;
            if (kind == 0) {
                z1 = st[0] > 20 ? 20 : (st[0] < -20 ? -20 : st[0]);
                z2 = st[1] > 20 ? 20 : (st[1] < -20 ? -20 : st[1]);
            } else {
                z1 = st[0] > 20 ? 20 : (st[0] < 0 ? 0 : st[0]);
                z2 = st[1] > 20 ? 20 : (st[1] < 0 ? 0 : st[1]);
            }
            m = st[3] != 0 ? 0 : st[2];
            const float* p = in + (size_t)(per * i) * stride;
            const float* r = p + stride;                           // M/S: the pair's R row
            const float mv = mvv[q];
            for (int n4 = nfram / 4, j = 0; n4--; j += 4) {
                if (kind == 0) {
                    const float t2 = z2 / 2;
                    for (int k = 0; k < 4; ++k) {
                        const float t1 = fabsf (p[j + k]) - t2;
                        z1 += w1 * (t1 - z1);
                    }
                    z2 += 4 * w1 * (z1 - z2);
                    if (z2 > m) m = z2;
                    tally (g, lim, edges, z2, c, a);
                } else {
                    z1 *= w3;
                    z2 *= w3;
                    for (int k = 0; k < 4; ++k) {
                        float t;
                        if (kind != 3) t = fabsf (p[j + k]);
                        else if (q == 0) t = mv * fabsf (p[j + k] + r[j + k]);
                        else t = mv * fabsf (p[j + k] - r[j + k]);
                        if (t > z1) z1 += w1 * (t - z1);
                        if (t > z2) z2 += w2 * (t - z2);
                    }
                    const float t = z1 + z2;
                    if (t > m) m = t;
                    tally (g, lim, edges, t, c, a);
                }
            }
            if (kind == 0) {
                if (!isfinite (z1)) { st[0] = 0; m = INFINITY; } else st[0] = z1;
                if (!isfinite (z2)) { st[1] = 0; m = INFINITY; } else st[1] = z2 + 1e-10f;
            } else {
                st[0] = z1 + 1e-10f;
                st[1] = z2 + 1e-10f;
            }
            st[2] = m;
            st[3] = 0;
        }
    }
}
