// _tpk_hist.cc — the distribution of the true-peak frames' and the K-meter groups' readings: the oracle of the true-peak / K-meter
// bank's histogram plane (b200m_tpk_hist_enable / b200m_tpk_hist_read).
//
// TEST INFRASTRUCTURE ONLY: compiled by tests/_tpk_hist.py into a temporary directory with the reference's float flags (SSE2
// arithmetic, no FMA contraction) and loaded by the tests; the product never links it.
//
// th_count counts readings with the rules of include/b200meters.h: the bin #{k : u >= e[k]} by a plain scan of the edge table,
// nonfinite, peak and the over runs against lim.  tests/_tpk_hist.py feeds it the true-peak frames' readings it forms from the
// reference build's resampler.
// th_km_run continues Kmeterdsp::process (jmeters/kmeterdsp.cc:56-103) of one meter from a copy of its z1 z2, taken from an oracle
// K-meter (_oracle.Kmeter.peek) just before the oracle runs the same frames: the clamp at call start, the "n /= 4" groups and the
// end-of-call scrub and bias.  After each group's z2 update it counts u = sqrtf (2 * z2), scanning the edges with u itself (not with
// the library's thresholds).  tests/_tpk_hist.py then checks the copy's z1 z2 bit for bit against the oracle's after its run.
#include <math.h>
#include <stddef.h>
#include <stdint.h>

struct Stats { uint64_t nonfinite, over_groups, overs, longest_over, run; float peak; uint32_t pad; };

static void tally (float u, float lim, const float* e, uint64_t* c, Stats* a)
{
    if (!isfinite (u)) { a->nonfinite += 1; return; }
    if (u > a->peak) a->peak = u;
    if (u >= lim) {
        a->over_groups += 1;
        if (a->run == 0) a->overs += 1;
        a->run += 1;
        if (a->run > a->longest_over) a->longest_over = a->run;
    } else a->run = 0;
    int k = 0;
    while (k < 241 && u >= e[k]) ++k;
    c[k] += 1;
}

// n readings of one row (non-finite ones included, as NaN or Inf)
extern "C" void th_count (const float* u, int n, float lim, const float* edges, uint64_t* counts /* [242] */, Stats* stats)
{
    for (int i = 0; i < n; ++i) tally (u[i], lim, edges, counts, stats);
}

// one K-meter over nfram frames; z = {z1, z2}, updated to the state the reference leaves
extern "C" void th_km_run (float omega, float lim, float* z, const float* p, int nfram, const float* edges, uint64_t* counts, Stats* stats)
{
    float s, z1 = z[0] > 50 ? 50 : (z[0] < 0 ? 0 : z[0]), z2 = z[1] > 50 ? 50 : (z[1] < 0 ? 0 : z[1]);
    for (int n = nfram / 4; n--;) {
        for (int k = 0; k < 4; ++k) {
            s = *p++;
            s *= s;
            z1 += omega * (s - z1);
        }
        z2 += 4 * omega * (z1 - z2);
        tally (sqrtf (2.0f * z2), lim, edges, counts, stats);
    }
    if (isnan (z1)) z1 = 0;
    if (isnan (z2)) z2 = 0;
    z[0] = z1 + 1e-20f;
    z[1] = z2 + 1e-20f;
}
