// _spec_ltas.cc — the long-term average spectrum (LTAS) of the spectrum plugin's per-frame band power: the oracle of the spectrum
// bank's LTAS plane (b200m_spec_ltas_enable / b200m_spec_ltas_read).
//
// TEST INFRASTRUCTURE ONLY: compiled by tests/_spec_ltas.py into a temporary directory with the reference's float flags (SSE2
// arithmetic, no FMA contraction) and loaded by the tests; the product never links it.
//
// sl_run continues each instance's 30 band-pass cascades from a copy of that instance's filter state, taken from an oracle
// spectr30 instance (_oracle.Spectr30.state) just before the oracle runs the same block.  Each band runs six transposed
// direct-form-II biquads in double (src/spectr.c:68-87) on (L + R) / 2.0f plus the alternating +-1e-12 bias, the band output v is
// rounded to float and s = v * v (src/spectrumlv2.c:221-226) is added to the band's double sum if it is finite, counting the frame.
// At the end it applies the run's scrub of non-finite states (:229-236), so tests/_spec_ltas.py can check the copy's end state
// bit for bit against the oracle's after its run: the sums are then those of the oracle's own per-frame power.
#include <math.h>
#include <stddef.h>
#include <stdint.h>

extern "C" void sl_run (int n, int nchan, const double* W /* [30][6][6] a0 a1 a2 b0 b1 b2 */, double* z /* [n][30][6][2] */,
                        const float* in, size_t stride, const int32_t* len /* [n] */, const int64_t* frames /* [n] */,
                        double* sums /* [n][30] */, uint64_t* counts /* [n][30] */)
{
    for (int i = 0; i < n; ++i) {
        if (len[i] <= 0) continue;                          // an instance that does not run keeps its state
        const float* l = in + (size_t)i * nchan * stride;
        const float* r = nchan == 2 ? l + stride : l;
        for (int b = 0; b < 30; ++b) {
            const double* w = W + b * 36;
            double* zb = z + ((size_t)i * 30 + b) * 12;
            for (int j = 0; j < len[i]; ++j) {
                const float x = nchan == 2 ? (l[j] + r[j]) / 2.0f : l[j];
                double y = x + (((frames[i] + j) & 1) == 0 ? 1e-12 : -1e-12);   // frame 0 of a fresh instance: +1e-12
                for (int s = 0; s < 6; ++s) {
                    const double* c = w + 6 * s;
                    double* zs = zb + 2 * s;
                    const double o = c[3] * y + zs[0];
                    zs[0] = c[4] * y - c[1] * o + zs[1];
                    zs[1] = c[5] * y - c[2] * o;
                    y = o;
                }
                const float v = (float)y;
                const float sq = v * v;
                if (isfinite (sq)) {
                    sums[i * 30 + b] += (double)sq;
                    counts[i * 30 + b] += 1;
                }
            }
            for (int k = 0; k < 12; ++k)
                if (!isfinite (zb[k])) zb[k] = 0;
        }
    }
}
