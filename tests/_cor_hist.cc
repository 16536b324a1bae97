// _cor_hist.cc — the distribution of Stcorrdsp's per-frame reading: the oracle of the correlation bank's histogram plane
// (b200m_cor_hist_enable / b200m_cor_hist_read).
//
// TEST INFRASTRUCTURE ONLY: compiled by tests/_cor_hist.py into a temporary directory with the reference's float flags (SSE2
// arithmetic, no FMA contraction) and loaded by the tests; the product never links it.
//
// ch_run continues each pair's five recurrences (jmeters/stcorrdsp.cc:58-62) from a copy of that pair's state, taken from an oracle
// Stcorrdsp bank (_oracle.Stcorr.peek) just before the oracle runs the same block.  After each frame it forms the reading
// r = zlr / sqrtf (zll * zrr + 1e-10f) (the read() formula, :79-82, on the in-loop state); if zll + zrr >= thr and r is finite, the
// frame adds 1 to bin clamp (floorf ((r + 1) * 100), 0, 199) and (double) r to the pair's sum.  At the end it applies process()'s
// scrub and bias (:65-75), so tests/_cor_hist.py can check the copy's end state bit for bit against the oracle's after its run.
#include <math.h>
#include <stddef.h>
#include <stdint.h>

extern "C" void ch_run (int n, float w1, float w2, float thr, float* state /* [n][5] zl zr zlr zll zrr */, const float* in,
                        size_t stride, int nfram, uint64_t* counts /* [n][200] */, double* sums /* [n] */)
{
    for (int i = 0; i < n; ++i) {
        const float* pl = in + (size_t)(2 * i) * stride;
        const float* pr = pl + stride;
        float* s = state + 5 * i;
        float zl = s[0], zr = s[1], zlr = s[2], zll = s[3], zrr = s[4];
        for (int j = 0; j < nfram; ++j) {
            zl += w1 * (pl[j] - zl) + 1e-20f;
            zr += w1 * (pr[j] - zr) + 1e-20f;
            zlr += w2 * (zl * zr - zlr);
            zll += w2 * (zl * zl - zll);
            zrr += w2 * (zr * zr - zrr);
            const float r = zlr / sqrtf (zll * zrr + 1e-10f);
            if (zll + zrr >= thr && isfinite (r)) {
                const float k = floorf ((r + 1.0f) * 100.0f);
                counts[(size_t)i * 200 + (int)(k < 0.0f ? 0.0f : (k > 199.0f ? 199.0f : k))] += 1;
                sums[i] += (double)r;
            }
        }
        if (!isfinite (zl)) zl = 0;
        if (!isfinite (zr)) zr = 0;
        if (!isfinite (zlr)) zlr = 0;
        if (!isfinite (zll)) zll = 0;
        if (!isfinite (zrr)) zrr = 0;
        s[0] = zl; s[1] = zr; s[2] = zlr + 1e-10f; s[3] = zll + 1e-10f; s[4] = zrr + 1e-10f;
    }
}
