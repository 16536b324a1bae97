// tpk.cu — true-peak (4x polyphase oversampler + PPM ballistics) and K-meter RMS bank.
//
// Replaces, for N mono channels at once, LV2M::TruePeakdsp (jmeters/truepeakdsp.cc:41-169) with its
// zita-resampler core (zita-resampler/resampler.cc:171-262, table resampler-table.cc:52-75) and
// LV2M::Kmeterdsp (jmeters/kmeterdsp.cc:47-162), as combined by dr14_run (src/dr14.c:391-394).
//
// Design (not the reference's ring-buffer walk): the resampler's steady state is a fixed
// 48-tap x 4-phase FIR over the last 48 inputs (SURVEY.md §8 a6), which is time-parallel, so a CTA
// stages [channels x chunk (+48 history)] tiles in shared memory with cp.async (8 x 256 for
// process_max, 16 x 64 for process) and every thread, staying on one channel row, produces 4 consecutive
// input positions x 4 phases = 16 outputs from a 52-float register window with the coefficients as
// instruction immediates.  Phase 0 of the table is a unit tap: under a proven magnitude guard it is the
// delayed input itself and is not evaluated (phase0_is_delay); rows of digital silence skip the FIR.
// The non-linear ballistics (truepeakdsp.cc:57-84), the K-meter recurrences and the DR-14 window sums
// are serial in time: lane roles on otherwise idle warps walk the |oversampled| / input tiles in shared
// memory while the other CTAs resident on the SM run their FIR phase.  The input is read from HBM
// exactly once for all meters.
// All arithmetic keeps the reference's operation order without FMA contraction: outputs are
// bit-identical to the reference build, not merely within tolerance.
#include <math.h>
#include <stdlib.h>
#include <algorithm>
#include "common.cuh"
#include "tpk_internal.cuh"
#include "ebu_kw.cuh"

namespace b200m {

constexpr int TPK_THREADS = 128;

__constant__ float c_tp_tab[120];           // zita table for hl=24, np=4, fr=1.0: [(np+1)][hl]

struct TpkParams {
    float w1, w2, w3, g;                    // TruePeakdsp::init (truepeakdsp.cc:153-157)
    float omega, fall; int hold;            // Kmeterdsp::init (kmeterdsp.cc:47-54), _fall for this n (:65-70)
    // tolerance mode, four K-meter steps at once: z1 <- z1 - kc4 z1 + (kq[0] s0 + kq[1] s1 + kq[2] s2 + kq[3] s3) with a = 1 - omega,
    // kq[i] = omega a^(3-i), kc4 = 1 - a^4 (all rounded once from double: the corner frequency keeps its 1e-7 relative accuracy)
    float kq[4], kc4;
};

struct TpkState {                           // SoA, one entry per channel
    float *hist;                            // [n_chan][48]: the 48 inputs preceding the next block
    float *tp_z1, *tp_z2, *tp_m, *tp_p; int *tp_res;
    float *km_z1, *km_z2, *km_rms, *km_peak, *km_fall; int *km_cnt, *km_fpp, *km_flag;
    unsigned* done_cnt;                     // CTAs of the running grid that reached their end (EBUr128 cycle, see the kernel's epilogue)
    float* hist_alt;                        // tpmax_kernel writes the next block's history here; the host swaps hist / hist_alt
    unsigned* blk_max;                      // [n_chan] running |v| maximum of the block being processed (float bits), tpmax_kernel
    unsigned* grp_cnt;                      // [n_chan] finished chunks of the channel group starting at this channel, tpmax_kernel
    float* tmp;                             // [7][n_chan] serial-meter state between the slabs of one block (tpbal_kernel): z1 z2 m p kz1 kz2 kt
    unsigned* sm_arr;                       // [256] process() CTAs that have arrived on each SM (phase stagger); NULL = no stagger
};

// The zita table depends only on (hl = 24, np = 4, fr = 1.0), not on the sample rate, so its 120 floats are universal
// constants.  They are restated here as literals (hex floats = the values libm produces for the formula in
// zita_table() below): with the tap loops fully unrolled the literals become FMUL immediates, which removes the ~50
// uniform constant loads per 16 outputs that the constant-bank form needs.  b200m_tpk_create compares the host-computed
// table with these literals bit for bit and falls back to the constant-bank kernels if they ever differ.
B200M_DEV float zita_lit (int i)
{
    switch (i) {
    case 0: return 0x1.0e8cc60000000p-65f;
    case 1: return -0x1.f4da040000000p-63f;
    case 2: return -0x1.1ecee20000000p-64f;
    case 3: return -0x1.9d9bde0000000p-62f;
    case 4: return 0x1.f84c660000000p-60f;
    case 5: return -0x1.5e4cb20000000p-60f;
    case 6: return -0x1.9321ea0000000p-60f;
    case 7: return -0x1.b534440000000p-59f;
    case 8: return 0x1.d2d4d80000000p-57f;
    case 9: return -0x1.bb55ce0000000p-58f;
    case 10: return -0x1.6e155a0000000p-57f;
    case 11: return -0x1.816e140000000p-57f;
    case 12: return 0x1.b8ff340000000p-55f;
    case 13: return -0x1.28f2680000000p-56f;
    case 14: return 0x1.62bccc0000000p-56f;
    case 15: return -0x1.9e31840000000p-56f;
    case 16: return 0x1.d96a6a0000000p-56f;
    case 17: return -0x1.092e9c0000000p-55f;
    case 18: return 0x1.237b360000000p-55f;
    case 19: return -0x1.3a9ac60000000p-55f;
    case 20: return 0x1.4da4960000000p-55f;
    case 21: return -0x1.5bd4640000000p-55f;
    case 22: return 0x1.6495740000000p-55f;
    case 23: return 0x1.0000000000000p+0f;
    case 24: return -0x1.d0758c0000000p-20f;
    case 25: return 0x1.74f3c80000000p-17f;
    case 26: return -0x1.21b2780000000p-15f;
    case 27: return 0x1.5cf90e0000000p-14f;
    case 28: return -0x1.6c77cc0000000p-13f;
    case 29: return 0x1.58b43e0000000p-12f;
    case 30: return -0x1.2e2f240000000p-11f;
    case 31: return 0x1.f29ba20000000p-11f;
    case 32: return -0x1.87672e0000000p-10f;
    case 33: return 0x1.26d2d00000000p-9f;
    case 34: return -0x1.ad12540000000p-9f;
    case 35: return 0x1.2f4f900000000p-8f;
    case 36: return -0x1.a293f80000000p-8f;
    case 37: return 0x1.1b24ca0000000p-7f;
    case 38: return -0x1.7912360000000p-7f;
    case 39: return 0x1.f0635e0000000p-7f;
    case 40: return -0x1.447e240000000p-6f;
    case 41: return 0x1.a7c41a0000000p-6f;
    case 42: return -0x1.168e760000000p-5f;
    case 43: return 0x1.7511480000000p-5f;
    case 44: return -0x1.03d1200000000p-4f;
    case 45: return 0x1.88e9740000000p-4f;
    case 46: return -0x1.6c09600000000p-3f;
    case 47: return 0x1.ccb95c0000000p-1f;
    case 48: return -0x1.1c1fd00000000p-20f;
    case 49: return 0x1.7106020000000p-17f;
    case 50: return -0x1.3e6cae0000000p-15f;
    case 51: return 0x1.927a360000000p-14f;
    case 52: return -0x1.b144fc0000000p-13f;
    case 53: return 0x1.a2f3160000000p-12f;
    case 54: return -0x1.75b1180000000p-11f;
    case 55: return 0x1.38a6c40000000p-10f;
    case 56: return -0x1.f0902a0000000p-10f;
    case 57: return 0x1.79a7c20000000p-9f;
    case 58: return -0x1.1509ce0000000p-8f;
    case 59: return 0x1.8a56220000000p-8f;
    case 60: return -0x1.11a21c0000000p-7f;
    case 61: return 0x1.73e48e0000000p-7f;
    case 62: return -0x1.f1065a0000000p-7f;
    case 63: return 0x1.47f5e80000000p-6f;
    case 64: return -0x1.ad4f620000000p-6f;
    case 65: return 0x1.183a9a0000000p-5f;
    case 66: return -0x1.6f76720000000p-5f;
    case 67: return 0x1.e924540000000p-5f;
    case 68: return -0x1.50663a0000000p-4f;
    case 69: return 0x1.ef2dda0000000p-4f;
    case 70: return -0x1.aa96140000000p-3f;
    case 71: return 0x1.4546e40000000p-1f;
    case 72: return -0x1.89a1500000000p-23f;
    case 73: return 0x1.5abb860000000p-18f;
    case 74: return -0x1.57d15a0000000p-16f;
    case 75: return 0x1.cbb6c20000000p-15f;
    case 76: return -0x1.ffab940000000p-14f;
    case 77: return 0x1.faa5820000000p-13f;
    case 78: return -0x1.cc49100000000p-12f;
    case 79: return 0x1.86d2e80000000p-11f;
    case 80: return -0x1.3a24580000000p-10f;
    case 81: return 0x1.e2abfe0000000p-10f;
    case 82: return -0x1.65134e0000000p-9f;
    case 83: return 0x1.ffdecc0000000p-9f;
    case 84: return -0x1.654aee0000000p-8f;
    case 85: return 0x1.e7f28c0000000p-8f;
    case 86: return -0x1.474f580000000p-7f;
    case 87: return 0x1.b124380000000p-7f;
    case 88: return -0x1.1bf13a0000000p-6f;
    case 89: return 0x1.72b7c40000000p-6f;
    case 90: return -0x1.e52f3e0000000p-6f;
    case 91: return 0x1.414ca20000000p-5f;
    case 92: return -0x1.b5509c0000000p-5f;
    case 93: return 0x1.3ad9d40000000p-4f;
    case 94: return -0x1.00d0b60000000p-3f;
    case 95: return 0x1.31e2140000000p-2f;
    case 96: return -0x0.0p+0f;
    case 97: return 0x1.0e8cc60000000p-65f;
    case 98: return -0x1.f4da040000000p-63f;
    case 99: return -0x1.1ecee20000000p-64f;
    case 100: return -0x1.9d9bde0000000p-62f;
    case 101: return 0x1.f84c660000000p-60f;
    case 102: return -0x1.5e4cb20000000p-60f;
    case 103: return -0x1.9321ea0000000p-60f;
    case 104: return -0x1.b534440000000p-59f;
    case 105: return 0x1.d2d4d80000000p-57f;
    case 106: return -0x1.bb55ce0000000p-58f;
    case 107: return -0x1.6e155a0000000p-57f;
    case 108: return -0x1.816e140000000p-57f;
    case 109: return 0x1.b8ff340000000p-55f;
    case 110: return -0x1.28f2680000000p-56f;
    case 111: return 0x1.62bccc0000000p-56f;
    case 112: return -0x1.9e31840000000p-56f;
    case 113: return 0x1.d96a6a0000000p-56f;
    case 114: return -0x1.092e9c0000000p-55f;
    case 115: return 0x1.237b360000000p-55f;
    case 116: return -0x1.3a9ac60000000p-55f;
    case 117: return 0x1.4da4960000000p-55f;
    case 118: return -0x1.5bd4640000000p-55f;
    case 119: return 0x1.6495740000000p-55f;
    default: return 0.0f;
    }
}
static const float h_zita_lit[120] = {0x1.0e8cc60000000p-65f, -0x1.f4da040000000p-63f, -0x1.1ecee20000000p-64f, -0x1.9d9bde0000000p-62f, 0x1.f84c660000000p-60f, -0x1.5e4cb20000000p-60f, -0x1.9321ea0000000p-60f, -0x1.b534440000000p-59f, 0x1.d2d4d80000000p-57f, -0x1.bb55ce0000000p-58f, -0x1.6e155a0000000p-57f, -0x1.816e140000000p-57f, 0x1.b8ff340000000p-55f, -0x1.28f2680000000p-56f, 0x1.62bccc0000000p-56f, -0x1.9e31840000000p-56f, 0x1.d96a6a0000000p-56f, -0x1.092e9c0000000p-55f, 0x1.237b360000000p-55f, -0x1.3a9ac60000000p-55f, 0x1.4da4960000000p-55f, -0x1.5bd4640000000p-55f, 0x1.6495740000000p-55f, 0x1.0000000000000p+0f, -0x1.d0758c0000000p-20f, 0x1.74f3c80000000p-17f, -0x1.21b2780000000p-15f, 0x1.5cf90e0000000p-14f, -0x1.6c77cc0000000p-13f, 0x1.58b43e0000000p-12f, -0x1.2e2f240000000p-11f, 0x1.f29ba20000000p-11f, -0x1.87672e0000000p-10f, 0x1.26d2d00000000p-9f, -0x1.ad12540000000p-9f, 0x1.2f4f900000000p-8f, -0x1.a293f80000000p-8f, 0x1.1b24ca0000000p-7f, -0x1.7912360000000p-7f, 0x1.f0635e0000000p-7f, -0x1.447e240000000p-6f, 0x1.a7c41a0000000p-6f, -0x1.168e760000000p-5f, 0x1.7511480000000p-5f, -0x1.03d1200000000p-4f, 0x1.88e9740000000p-4f, -0x1.6c09600000000p-3f, 0x1.ccb95c0000000p-1f, -0x1.1c1fd00000000p-20f, 0x1.7106020000000p-17f, -0x1.3e6cae0000000p-15f, 0x1.927a360000000p-14f, -0x1.b144fc0000000p-13f, 0x1.a2f3160000000p-12f, -0x1.75b1180000000p-11f, 0x1.38a6c40000000p-10f, -0x1.f0902a0000000p-10f, 0x1.79a7c20000000p-9f, -0x1.1509ce0000000p-8f, 0x1.8a56220000000p-8f, -0x1.11a21c0000000p-7f, 0x1.73e48e0000000p-7f, -0x1.f1065a0000000p-7f, 0x1.47f5e80000000p-6f, -0x1.ad4f620000000p-6f, 0x1.183a9a0000000p-5f, -0x1.6f76720000000p-5f, 0x1.e924540000000p-5f, -0x1.50663a0000000p-4f, 0x1.ef2dda0000000p-4f, -0x1.aa96140000000p-3f, 0x1.4546e40000000p-1f, -0x1.89a1500000000p-23f, 0x1.5abb860000000p-18f, -0x1.57d15a0000000p-16f, 0x1.cbb6c20000000p-15f, -0x1.ffab940000000p-14f, 0x1.faa5820000000p-13f, -0x1.cc49100000000p-12f, 0x1.86d2e80000000p-11f, -0x1.3a24580000000p-10f, 0x1.e2abfe0000000p-10f, -0x1.65134e0000000p-9f, 0x1.ffdecc0000000p-9f, -0x1.654aee0000000p-8f, 0x1.e7f28c0000000p-8f, -0x1.474f580000000p-7f, 0x1.b124380000000p-7f, -0x1.1bf13a0000000p-6f, 0x1.72b7c40000000p-6f, -0x1.e52f3e0000000p-6f, 0x1.414ca20000000p-5f, -0x1.b5509c0000000p-5f, 0x1.3ad9d40000000p-4f, -0x1.00d0b60000000p-3f, 0x1.31e2140000000p-2f, -0x0.0p+0f, 0x1.0e8cc60000000p-65f, -0x1.f4da040000000p-63f, -0x1.1ecee20000000p-64f, -0x1.9d9bde0000000p-62f, 0x1.f84c660000000p-60f, -0x1.5e4cb20000000p-60f, -0x1.9321ea0000000p-60f, -0x1.b534440000000p-59f, 0x1.d2d4d80000000p-57f, -0x1.bb55ce0000000p-58f, -0x1.6e155a0000000p-57f, -0x1.816e140000000p-57f, 0x1.b8ff340000000p-55f, -0x1.28f2680000000p-56f, 0x1.62bccc0000000p-56f, -0x1.9e31840000000p-56f, 0x1.d96a6a0000000p-56f, -0x1.092e9c0000000p-55f, 0x1.237b360000000p-55f, -0x1.3a9ac60000000p-55f, 0x1.4da4960000000p-55f, -0x1.5bd4640000000p-55f, 0x1.6495740000000p-55f};

// Phase 0 of the zita table is a unit tap (tab[23] = 1.0f) among 46 taps of magnitude <= 1.73 * 2^-55 (plus one -0.0f);
// the 46 magnitudes sum to S = 7.7035e-16.  Its output is therefore x[k-24] itself whenever the tiny products and the
// +-1e-20f bias are too small to move any partial sum off x[k-24].  Sufficient condition used here, for the window
// maximum M >= max |w[j]| (NaN-propagating; taken over the whole chunk row, see row_absmax):
//     |x| > 1.25e-7 * M + 1e-12        (then x is normal and M finite)       or       M == 0 (silent row: output +0)
// Proof: the unit tap is the last pair (i = 23).  Every partial sum before it is bounded by
// A = (1e-20 + S * M) * (1 + 2^-18) < 1.0001e-20 + 7.71e-16 * M, and so is the other product of the last pair.  With
// 2^e <= |x| < 2^(e+1): A < |x| * 2^-26 < 2^(e-25) = half of the smallest gap next to x, so fl(x + tiny) = x,
// fl(acc + x) = x and fl(x - 1e-20f) = x under round-to-nearest.  |x| * 2^-26 > A  <=>  |x| > 6.72e-13 + 5.18e-8 * M;
// the guard's constants leave 2.4x / 1.5x of margin over that, far more than the rounding of the guard itself.
// Non-finite samples make M NaN/Inf and fail the test, so such windows take the full evaluation (NaN/Inf propagate
// exactly as in the reference).  b200m_tpk_create enables the shortcut only after checking tab[23] == 1 and S against
// the table it actually computed.  Checked offline on 2e8 random / adversarial windows (0 mismatches) and by
// tests/test_tpk_gpu.py::test_phase0_guard_* on both sides of the guard.
B200M_DEV float max3_abs_nan (float a, float b, float c)             // max (|a|, |b|, |c|), NaN if any operand is NaN
{
    float d;
    asm ("max.NaN.f32 %0, %1, %2;" : "=f"(d) : "f"(fabsf (a)), "f"(fabsf (b)));
    asm ("max.NaN.f32 %0, %0, %1;" : "+f"(d) : "f"(fabsf (c)));
    return d;
}

// |x| maximum (NaN-propagating) of one shared-memory row of NV float4, computed by the SEG lanes of the warp that work on
// that row; every lane of the segment returns the same M.  M covers more than the 48 taps a sample needs (the whole
// chunk + its 48-sample prefix), which only makes the guard more conservative.
template <int SEG, int NV>
B200M_DEV float row_absmax (const float4* __restrict__ row, int lane)
{
    float mx = 0.0f;
#pragma unroll
    for (int j0 = 0; j0 < NV; j0 += SEG) {
        const int j = j0 + (lane & (SEG - 1));
        if (j0 + SEG <= NV || j < NV) { const float4 v = row[j]; mx = max3_abs_nan (max3_abs_nan (v.x, v.y, v.z), v.w, mx); }
    }
    // mx >= +0 or NaN (0x7fffffff): unsigned order == float order with NaN on top
    const unsigned segmask = SEG == 32 ? 0xffffffffu : (((1u << SEG) - 1u) << (lane & ~(SEG - 1)));
    return __uint_as_float (__reduce_max_sync (segmask, __float_as_uint (mx)));
}

B200M_DEV bool phase0_is_delay (const float4 x, const float M)
{
    // M == 0: the whole row is +-0 and the full evaluation yields (1e-20f + 0) - 1e-20f = +0 (digital silence stays fast)
    const float thr = __fadd_rn (__fmul_rn (M, 1.25e-7f), 1e-12f);
    return (fabsf (x.x) > thr && fabsf (x.y) > thr && fabsf (x.z) > thr && fabsf (x.w) > thr) || M == 0.0f;
}

// 16 outputs (4 input positions x 4 phases) from a 52-sample window; w[j] = x[kb-48+j].
// out[4k+ph] = (1e-20f + sum_i (x[k-47+i]*c1[i] + x[k-i]*c2[i])) - 1e-20f, pair-sum first, i ascending
// (resampler.cc:213-230 with c1 = ctab + hl*ph, c2 = ctab + hl*(np-ph)).
// `full0` (warp-uniform) = evaluate phase 0 as well; otherwise phase 0 is the proven pure delay (see above).  The
// full evaluation re-reads its window from shared memory (`xw`, volatile so that the loads are not merged with the
// ones feeding `w`): keeping `w` alive across the branch instead costs ~40 registers and a third of the occupancy.
B200M_DEV float lds_volatile (const float* p)
{
    float v;
    asm volatile ("ld.volatile.shared.f32 %0, [%1];" : "=f"(v) : "r"((unsigned)__cvta_generic_to_shared (p)));
    return v;
}

template <bool IMM>
B200M_DEV void fir16 (const float (&w)[52], const float* xw, float (&o)[16], const bool full0)
{
    float acc[16];
#pragma unroll
    for (int a = 0; a < 16; ++a) acc[a] = 1e-20f;
#pragma unroll
    for (int i = 0; i < 24; ++i) {
#pragma unroll
        for (int ph = 1; ph < 4; ++ph) {
            const float c1 = IMM ? zita_lit (24 * ph + i) : c_tp_tab[24 * ph + i];
            const float c2 = IMM ? zita_lit (24 * (4 - ph) + i) : c_tp_tab[24 * (4 - ph) + i];
#pragma unroll
            for (int r = 0; r < 4; ++r)
                acc[4 * r + ph] = __fadd_rn (acc[4 * r + ph], __fadd_rn (__fmul_rn (w[r + i + 1], c1), __fmul_rn (w[r + 48 - i], c2)));
        }
    }
#pragma unroll
    for (int a = 0; a < 16; ++a) o[a] = __fsub_rn (acc[a], 1e-20f);
#pragma unroll
    for (int r = 0; r < 4; ++r) o[4 * r] = __fadd_rn (w[r + 24], 0.0f);      // x for x != 0; +0 for the all-zero row (-0 + 0 = +0)
    if (full0) {
        // two sliding 4-sample windows: lo = x[i+1 .. i+4], hi = x[48-i .. 51-i]; one new sample each per tap pair
        float a0[4] = {1e-20f, 1e-20f, 1e-20f, 1e-20f};
        float lo[4], hi[4];
#pragma unroll
        for (int r = 0; r < 3; ++r) { lo[r + 1] = lds_volatile (xw + r + 1); hi[r] = lds_volatile (xw + 49 + r); }
#pragma unroll
        for (int i = 0; i < 24; ++i) {
            const float c1 = IMM ? zita_lit (i) : c_tp_tab[i];
            const float c2 = IMM ? zita_lit (96 + i) : c_tp_tab[96 + i];
#pragma unroll
            for (int r = 0; r < 3; ++r) { lo[r] = lo[r + 1]; hi[3 - r] = hi[2 - r]; }
            lo[3] = lds_volatile (xw + i + 4); hi[0] = lds_volatile (xw + 48 - i);
#pragma unroll
            for (int r = 0; r < 4; ++r)
                a0[r] = __fadd_rn (a0[r], __fadd_rn (__fmul_rn (lo[r], c1), __fmul_rn (hi[r], c2)));
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) o[4 * r] = __fsub_rn (a0[r], 1e-20f);
    }
}

// ---- tolerance mode (B200M_PREC_FMA) ------------------------------------------------------------------------------------
// north_star asks for float outputs within +-1e-4 dB of the reference and bit-exact INTEGER results; dBTP and the true-peak
// ballistics feed no histogram, so the 4x FIR may round differently from the reference's unfused SSE2 sequence as long as it
// stays inside that tolerance.  fir16_fma is the same 48-tap x 4-phase filter with
//   * phase 0 = the delayed input itself (its other 46 taps weigh 7.7e-16 in total: 7e-15 dB),
//   * phases 1..3 accumulated with FFMA from 0 (no +-1e-20f bias), and
//   * (SYM) the table's symmetry: phase 3 is phase 1 mirrored and phase 2 is its own mirror, so with s = a + b, d = a - b of a
//     tap pair (a = x[k-47+i], b = x[k-i]):  P = ph1 + ph3 = sum s (c1 + c3),  Q = ph1 - ph3 = sum d (c1 - c3),  ph2 = sum s c2
//     -> 2 FADD + 3 FFMA per tap pair instead of 6 FFMA: 120 fp32 instructions per input sample (exact mode: 288 + guard).
// Measured deviation from the reference on white noise: see tests/test_tpk_gpu.py::test_fma_mode_within_tolerance
// (|delta| <= 2e-6 of the block peak, i.e. <= 2e-5 dB on the peak reading).
#ifndef B200M_TPK_SYM
#define B200M_TPK_SYM 1
#endif
B200M_DEV float fmax3 (float a, float b, float c)                    // fmaxf (fmaxf (a, b), c): NaN operands ignored
{
    return fmaxf (fmaxf (a, b), c);
}

B200M_DEV float max3_abs (float a, float b, float c)                 // max (|a|, |b|, |c|), NaN operands ignored like fmaxf
{
    return fmaxf (fmaxf (fabsf (a), fabsf (b)), fabsf (c));
}

#if B200M_TPK_SYM
template <bool IMM>
B200M_DEV void fir_pqr (const float (&w)[52], float (&P)[4], float (&Q)[4], float (&R)[4])
{
#pragma unroll
    for (int r = 0; r < 4; ++r) { P[r] = 0.0f; Q[r] = 0.0f; R[r] = 0.0f; }
#pragma unroll
    for (int i = 0; i < 24; ++i) {
        const float t1 = IMM ? zita_lit (24 + i) : c_tp_tab[24 + i];
        const float t3 = IMM ? zita_lit (72 + i) : c_tp_tab[72 + i];
        const float t2 = IMM ? zita_lit (48 + i) : c_tp_tab[48 + i];
        const float cs = t1 + t3, cd = t1 - t3;                 // folded at compile time when IMM
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const float a = w[r + i + 1], b = w[r + 48 - i];
            const float sm = __fadd_rn (a, b), df = __fsub_rn (a, b);
            P[r] = fmaf (sm, cs, P[r]);
            Q[r] = fmaf (df, cd, Q[r]);
            R[r] = fmaf (sm, t2, R[r]);
        }
    }
}

// running maxima of the 4 x `nvalid` outputs without forming phases 1 and 3: max (|ph1|, |ph3|) = (|P| + |Q|) / 2 exactly (one of
// P + Q, P - Q is the sum of the magnitudes; rounding is sign-symmetric), so `vb` collects |P| + |Q| and the caller halves it once
template <bool IMM>
B200M_DEV void fir16_fma_max (const float (&w)[52], int nvalid, float& va, float& vb)
{
    float P[4], Q[4], R[4];
    fir_pqr<IMM> (w, P, Q, R);
#pragma unroll
    for (int r = 0; r < 4; ++r)
        if (r < nvalid) { va = max3_abs (va, w[r + 24], R[r]); vb = fmaxf (vb, __fadd_rn (fabsf (P[r]), fabsf (Q[r]))); }
}
#endif

template <bool IMM>
B200M_DEV void fir16_fma (const float (&w)[52], float (&o)[16])
{
#if B200M_TPK_SYM
    float P[4], Q[4], R[4];
    fir_pqr<IMM> (w, P, Q, R);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        o[4 * r] = w[r + 24];
        o[4 * r + 1] = __fmul_rn (0.5f, __fadd_rn (P[r], Q[r]));
        o[4 * r + 2] = R[r];
        o[4 * r + 3] = __fmul_rn (0.5f, __fsub_rn (P[r], Q[r]));
    }
#else
    float acc[16];
#pragma unroll
    for (int a = 0; a < 16; ++a) acc[a] = 0.0f;
#pragma unroll
    for (int i = 0; i < 24; ++i) {
#pragma unroll
        for (int ph = 1; ph < 4; ++ph) {
            const float c1 = IMM ? zita_lit (24 * ph + i) : c_tp_tab[24 * ph + i];
            const float c2 = IMM ? zita_lit (24 * (4 - ph) + i) : c_tp_tab[24 * (4 - ph) + i];
#pragma unroll
            for (int r = 0; r < 4; ++r) acc[4 * r + ph] = fmaf (w[r + i + 1], c1, fmaf (w[r + 48 - i], c2, acc[4 * r + ph]));
        }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) { o[4 * r] = w[r + 24]; o[4 * r + 1] = acc[4 * r + 1]; o[4 * r + 2] = acc[4 * r + 2]; o[4 * r + 3] = acc[4 * r + 3]; }
#endif
}

// Tile geometry: CH channels x TC input samples per chunk.  process_max (no serial true-peak lane) uses
// <8,256>: 2048 CTAs for 16384 channels, 8 resident per SM.  process() uses <16,64>: the ballistics warp then runs
// 16 channels x {z1 filter, z2 filter} = 32 busy lanes (the two one-pole attack filters are independent until
// the per-sample m = max (m, z1 + z2), which costs one shuffle), so the serial part issues ~1/4 of the
// instructions it would with one channel per lane.
// shared-memory geometry of tpk_kernel.  Row pitch of the x tile: lanes of a quarter warp that read 16-byte groups of DIFFERENT rows
// must land in different banks; with LPR = 128 / CH lanes per row that needs a pitch of 4 * LPR mod 32 floats when LPR < 8.
template <int CH, int TC, bool BAL>
struct TpkGeom {
    static constexpr int XP = (CH == 64) ? (48 + TC + 4 + 31) / 32 * 32 + 8 : 48 + TC + 4;
    static constexpr int OP = 4 * TC + 4;
    static constexpr size_t BYTES = (size_t)(2 * CH * XP + (BAL ? CH * OP : 4)) * sizeof (float);
};

// EBUr128 epilogue (src/ebulv2.cc:227-230,360-367), called by a whole warp whose lanes hold consecutive channels cc = c0 + lane
// (a true-peak group: lanes 0..7; a fused slab: all 32; own: cc is one of the kernel's channels) and their read() mm (returns _m,
// sets _res, truepeakdsp.cc:133-138).  HOLD = nch = 1, 2, 4: the warp holds whole instances (c0 is a multiple of nch); the
// instance's first lane takes t = the largest of its channels' reads (they are >= +0 and never NaN, so the order of the
// comparisons does not matter) and holds coef_to_db (t).  HOLD = 0 (nch = 3, 5): every read goes to r.lin[cc] for r128_hold_kernel.
// The kernels with this epilogue take HOLD as a template parameter (r128_hold_of picks it): the fold is then one shuffle and
// shifts for stereo, with no run-time channel count in the epilogue's code.
template <int HOLD>
B200M_DEV void r128_group_hold (const R128Hold& r, const TpkState& st, float mm, int cc, bool own)
{
    static_assert (HOLD == 0 || HOLD == 1 || HOLD == 2 || HOLD == 4, "instances must not leave a group");
    if (own) st.tp_res[cc] = 1;
    if constexpr (HOLD == 0) {
        if (own) r.lin[cc] = mm;
    } else {
        float t = mm;
#pragma unroll
        for (int o = 1; o < HOLD; o <<= 1) { const float b = __shfl_xor_sync (0xffffffffu, t, o); t = t > b ? t : b; }
        if (own && (unsigned)cc % HOLD == 0) r128_hold (r.tpmax + (unsigned)cc / HOLD, t);
    }
}
// the HOLD instantiation for a launch: 2 (the stereo code) when the launch has no EBUr128 epilogue
static inline int r128_hold_of (const R128Hold& r) { return !r.tpmax ? 2 : r.lin ? 0 : r.nch; }

template <int CH, int TC, bool TP, bool TPMAX, bool KM, bool IMM, bool DR, bool FMA = false>
__global__ void __launch_bounds__ (TPK_THREADS)
tpk_kernel (const float* __restrict__ in, size_t stride, int c_first, int n_chan, int nfram, int aligned, int elide0, TpkParams prm,
            TpkState st, float* __restrict__ dbg, R128Hold r128, TpkDr dr)
{
    // processes channels [c_first, n_chan): `n_chan` is the END of the slice (absolute channel index)
    constexpr int XP = TpkGeom<CH, TC, TP && !TPMAX>::XP;   // x row pitch (floats): 16-byte multiple
    constexpr int OP = 4 * TC + 4;                // |out| row pitch
    constexpr int GPC = TC / 4;                   // 4-sample groups per channel per chunk
    constexpr bool BAL = TP && !TPMAX;
    // ballistics lanes come in groups of 16 channels x 2 filters = one warp: a 16-channel CTA has one such warp (the other three do the
    // K-meter / DR roles or idle during the serial phase), a 64-channel CTA ("wide") keeps ALL four warps busy in the serial phase.
    // 87 KB of shared memory per CTA leave two CTAs = eight warps per SM, too few to hide the FIR's latencies (the 16-channel form
    // keeps seven CTAs resident and lets other CTAs' FIR phases run under a CTA's serial phase; its DR form takes 94 registers and
    // keeps five, measured faster than the same code bounded to seven, meters.lv2_b200/host/dr14_run_cost.py).  Kept opt-in,
    // bit-identical, tested.
    static_assert (!BAL || CH == 16 || CH == 64, "split ballistics lanes assume 16 channels per warp");
    constexpr bool ALLW = BAL && CH == 64;
    constexpr int LPR = TPK_THREADS / CH;         // lanes that share one channel row in the FIR phase (an aligned lane group)
    static_assert (CH <= 64 && TPK_THREADS % CH == 0 && LPR <= 32 && GPC % LPR == 0, "tile geometry");
    extern __shared__ __align__ (16) float tpk_smem[];        // xs[2][CH][XP], then ob[BAL ? CH : 1][BAL ? OP : 4]
    float (*xs)[CH][XP] = reinterpret_cast<float (*)[CH][XP]> (tpk_smem);
    float (*ob)[BAL ? OP : 4] = reinterpret_cast<float (*)[BAL ? OP : 4]> (tpk_smem + 2 * CH * XP);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int c0 = c_first + blockIdx.x * CH;
    // Chunk schedule.  Co-resident CTAs of process() start together and would run their FIR phases (issue-bound, every warp busy) and
    // their serial phases (latency-bound, one or two warps busy) in lock step, leaving the SM idle through every serial phase.  Every
    // second CTA to arrive on an SM therefore shortens its FIRST chunk to TC / 2 samples, which shifts all its later phases by half a
    // period against its neighbours'.  Chunk boundaries stay multiples of 4 samples (the K-meter's stride) and every per-sample
    // operation is unchanged, so the results do not depend on which CTAs shift.
    // Opt-in (B200M_TPK_STAGGER=1), covered by tests.
    __shared__ int s_lead;
    if (BAL && st.sm_arr != nullptr) {
        if (tid == 0) {
            unsigned smid; asm ("mov.u32 %0, %%smid;" : "=r"(smid));
            s_lead = (atomicAdd (st.sm_arr + (smid & 255u), 1u) & 1u) ? TC / 2 : 0;
        }
        __syncthreads ();
    }
    const int lead = (BAL && st.sm_arr != nullptr) ? s_lead : 0;
    const int nchunks = (nfram + lead + TC - 1) / TC;
    auto chunk_start = [&] (int c) { return max (0, c * TC - lead); };
    auto chunk_end = [&] (int c) { return min (nfram, (c + 1) * TC - lead); };

    auto load_chunk = [&] (int c, int buf) {
        if (c < nchunks) {
            const int s0 = chunk_start (c);
            if (aligned) {
#pragma unroll
                for (int idx = tid; idx < CH * GPC; idx += TPK_THREADS) {      // CH rows x GPC 16-byte pieces
                    const int r = idx / GPC, c4 = (idx % GPC) * 4;
                    const int ch = min (c0 + r, n_chan - 1);
                    const int left = (nfram - (s0 + c4)) * 4;
                    const int nb = left >= 16 ? 16 : (left > 0 ? left : 0);
                    cp_async16 (&xs[buf][r][48 + c4], nb ? in + (size_t)ch * stride + s0 + c4 : in, nb);
                }
            } else {
                for (int idx = tid; idx < CH * TC; idx += TPK_THREADS) {
                    const int r = idx / TC, cc = idx % TC;
                    const int ch = min (c0 + r, n_chan - 1);
                    const bool ok = (s0 + cc) < nfram;
                    cp_async4 (&xs[buf][r][48 + cc], ok ? in + (size_t)ch * stride + s0 + cc : in, ok ? 4 : 0);
                }
            }
        }
        cp_async_commit ();
    };

    // history -> xs[0][.][0..47]
    for (int idx = tid; idx < CH * 48; idx += TPK_THREADS) {
        const int r = idx / 48, j = idx % 48;
        xs[0][r][j] = TP ? st.hist[(size_t)min (c0 + r, n_chan - 1) * 48 + j] : 0.0f;
    }
    load_chunk (0, 0);

    // serial lanes.  role 0: true-peak ballistics, lane = filter * 16 + channel.  role 1: K-meter, lane = channel.
    // the serial roles rotate over the CTA's warps with blockIdx: warp w of every CTA lives on SM sub-partition w % 4, so a
    // fixed role assignment would pile all ballistics work (18 % of the instructions) onto sub-partition 0
    const int wrole = (warp + blockIdx.x) & 3;
    const int wbase = ALLW ? 16 * warp : 0;               // wide CTA: warp w serves channels 16 w .. 16 w + 15 in every serial role
    const bool is_tp = BAL && (ALLW || wrole == 0);
    const int tch = lane & 15, filt = lane >> 4;
    const bool is_km = KM && (ALLW ? lane < 16 : (wrole == 1 && lane < CH));
    const int srow = wbase + (is_tp ? tch : lane);         // tile row of this lane's serial channel
    const int chs = min (c0 + srow, n_chan - 1);
    const bool live = (c0 + srow) < n_chan;
    float z = 0, m = 0, p = 0, wf = 0; int res = 0;
    float kz1 = 0, kz2 = 0, kt = 0;
    if (is_tp) {
        res = st.tp_res[chs];
        m = res ? 0.0f : st.tp_m[chs];                                  // truepeakdsp.cc:52-55
        p = res ? 0.0f : st.tp_p[chs];
        const float a = filt ? st.tp_z2[chs] : st.tp_z1[chs];
        z = a > 20 ? 20 : (a < 0 ? 0 : a);
        wf = filt ? prm.w2 : prm.w1;
    }
    if (is_km) {
        const float a = st.km_z1[chs], b = st.km_z2[chs];               // kmeterdsp.cc:74-75
        kz1 = a > 50 ? 50 : (a < 0 ? 0 : a);
        kz2 = b > 50 ? 50 : (b < 0 ? 0 : b);
    }
    // role 2 (idle otherwise while the serial lanes run): DR-14 sums, lane = channel
    const bool dr_warp = DR && BAL && KM && dr.rms_sum != nullptr && (ALLW || wrole == 2);
    const int drow = wbase + (lane & 15);
    const int dch = min (c0 + drow, n_chan - 1);
    const bool dr_live = dr_warp && lane < 16 && (c0 + drow) < n_chan;
    float drs = 0, drp = 0; int dcut = -1;
    if (dr_warp) { drs = dr.rms_sum[dch]; drp = dr.peak_cur[dch]; dcut = tpk_dr_cut (dr, dch / dr.nch, nfram); }
    // the first window end of the warp's lanes in this block (each lane's instance has its own); the warp reaches it together, so
    // the silence test's partner exchange is a convergent shuffle
    int wcut = dr_warp ? __reduce_min_sync (0xffffffffu, dcut >= 0 ? dcut : INT_MAX) : INT_MAX;
    float vmax = 0.0f;                                                    // process_max: plain running max (:109-122), per FIR lane
    const int km_n = (nfram / 4) * 4;                                     // "n /= 4" drops n mod 4 samples (:79)

    for (int c = 0; c < nchunks; ++c) {
        const int buf = c & 1;
        const int s0 = chunk_start (c);
        const int len = chunk_end (c) - s0;
        cp_async_wait<0> ();
        __syncthreads ();                                   // chunk c (and its 48-sample prefix) is in xs[buf]
        // prefix of the next chunk = last 48 samples of this one; start the next load
        for (int idx = tid; idx < CH * 48; idx += TPK_THREADS) {
            const int r = idx / 48, j = idx % 48;
            xs[buf ^ 1][r][j] = xs[buf][r][len + j];
        }
        load_chunk (c + 1, buf ^ 1);

        if (TP) {
            // FIR phase: a thread stays on channel row r = tid / LPR for the whole block and takes the groups q = ql + k * LPR
            // of 4 consecutive inputs (consecutive lanes -> consecutive 16-byte groups: conflict-free LDS.128)
            const int r = tid / LPR, ql = tid % LPR;
            float M = 0.0f;
            if (elide0) M = row_absmax<LPR, 12 + GPC> (reinterpret_cast<const float4*> (&xs[buf][r][0]), lane);
            // digital silence on every row this warp works on (chunk + its 48-sample prefix all +-0): each of the 4 phases is
            // (1e-20f + 0) - 1e-20f = +0, so the FIR is skipped altogether (idle channels of a large bank cost no arithmetic)
            const bool silent_rows = elide0 && __all_sync (0xffffffffu, M == 0.0f);
            if (silent_rows) {
                // outputs are all +0: nothing to add to a running max; process() still needs its |out| tile, the debug tap its zeros
                for (int q = ql; q < GPC && 4 * q < len; q += LPR) {
                    if (BAL) {
                        float4* d = reinterpret_cast<float4*> (&ob[BAL ? r : 0][0]);
#pragma unroll
                        for (int i = 0; i < 4; ++i) d[BAL ? i * GPC + q : 0] = make_float4 (0.0f, 0.0f, 0.0f, 0.0f);
                    }
                    if (dbg && (c0 + r) < n_chan) {
                        float4* d = reinterpret_cast<float4*> (dbg + (size_t)(c0 + r) * (4 * B200M_MAX_BLOCK) + 4 * (s0 + 4 * q));
#pragma unroll
                        for (int i = 0; i < 4; ++i) d[i] = make_float4 (0.0f, 0.0f, 0.0f, 0.0f);
                    }
                }
            } else
#pragma unroll 1
            for (int q = ql; q < GPC; q += LPR) {
                const bool act = 4 * q < len;
                // phase 0 degenerates to a delay for every lane of the warp?  (one vote keeps the branch warp-uniform;
                // lanes beyond a short block's end vote yes)
                bool full0 = !FMA;
                if (!FMA && elide0) {
                    const float4 xm = *reinterpret_cast<const float4*> (&xs[buf][r][act ? 4 * q + 24 : 0]);   // the 4 unit-tap samples
                    full0 = !__all_sync (0xffffffffu, !act || phase0_is_delay (xm, M));
                }
                if (act) {
                    float w[52];
                    const float4* xr = reinterpret_cast<const float4*> (&xs[buf][r][4 * q]);
#pragma unroll
                    for (int i = 0; i < 13; ++i) { const float4 v = xr[i]; w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w; }
                    float o[16];
                    if (FMA) fir16_fma<IMM> (w, o); else fir16<IMM> (w, &xs[buf][r][4 * q], o, full0);
                    if (dbg && (c0 + r) < n_chan) {
                        float4* d = reinterpret_cast<float4*> (dbg + (size_t)(c0 + r) * (4 * B200M_MAX_BLOCK) + 4 * (s0 + 4 * q));
#pragma unroll
                        for (int i = 0; i < 4; ++i) d[i] = make_float4 (o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
                    }
                    if (TPMAX) {
                        // positions beyond len inside the last group come from zero-filled input: exclude them.
                        // fmaxf == the reference's `if (v > m) m = v` here: m is never NaN and a NaN v leaves it unchanged
#pragma unroll
                        for (int i = 0; i < 4; ++i)
                            if (4 * q + i < len)
                                vmax = fmaxf (fmaxf (vmax, fmaxf (fabsf (o[4 * i]), fabsf (o[4 * i + 1]))), fmaxf (fabsf (o[4 * i + 2]), fabsf (o[4 * i + 3])));
                    } else {
                        // the 4 outputs of input sample 4q+i live at float4 slot i*GPC + q: consecutive lanes (q) store
                        // consecutive float4 -> conflict-free STS.128; the ballistics lane un-swizzles when it reads
                        float4* d = reinterpret_cast<float4*> (&ob[BAL ? r : 0][0]);
#pragma unroll
                        for (int i = 0; i < 4; ++i)
                            d[BAL ? i * GPC + q : 0] = make_float4 (fabsf (o[4 * i]), fabsf (o[4 * i + 1]), fabsf (o[4 * i + 2]), fabsf (o[4 * i + 3]));
                    }
                }
            }
        }
        if (BAL) __syncthreads ();                          // |out| tile complete

        if (is_tp) {
            // PPM ballistics over the 4*len oversampled magnitudes (truepeakdsp.cc:57-84); this lane owns one of the
            // two attack filters of channel tch.  Samples are taken four at a time (the tile's float4 slots i * GPC + g of group g
            // sit at constant offsets from one moving base, and the next group's loads are issued before this group's chain).
            const float4* b4 = reinterpret_cast<const float4*> (&ob[BAL ? wbase + tch : 0][0]);
            // tolerance mode: z <- max (z, (1 - w) z + w v) is `if (v > z) z += w (v - z)` in real arithmetic; with w' = 1 - fl (1 - w)
            // the pair (1 - w, w') sums to one exactly, so a settled filter sits on its input, and the time constant moves by < 2e-6
            // relative.  Two dependent instructions per oversampled value instead of four: 41 cycles per input sample instead of 102.
            const float omw = __fsub_rn (1.0f, wf), wq = __fsub_rn (1.0f, omw), omw3 = __fmul_rn (omw, prm.w3);
            auto step = [&] (const float4 v4) {
                if (FMA) {
                    const float zd = __fmul_rn (z, prm.w3);
                    z = fmaxf (zd, fmaf (omw3, z, __fmul_rn (wq, v4.x)));
                    z = fmaxf (z, fmaf (omw, z, __fmul_rn (wq, v4.y)));
                    z = fmaxf (z, fmaf (omw, z, __fmul_rn (wq, v4.z)));
                    z = fmaxf (z, fmaf (omw, z, __fmul_rn (wq, v4.w)));
                } else {
                    z = __fmul_rn (z, prm.w3);
                    if (v4.x > z) z = __fadd_rn (z, __fmul_rn (wf, __fsub_rn (v4.x, z)));
                    if (v4.y > z) z = __fadd_rn (z, __fmul_rn (wf, __fsub_rn (v4.y, z)));
                    if (v4.z > z) z = __fadd_rn (z, __fmul_rn (wf, __fsub_rn (v4.z, z)));
                    if (v4.w > z) z = __fadd_rn (z, __fmul_rn (wf, __fsub_rn (v4.w, z)));
                }
                // == four times `if (v > p) p = v`: p is never NaN, NaN values leave it unchanged (3-input FMNMX ignores NaN operands)
                p = fmax3 (p, fmax3 (v4.x, v4.y, v4.z), v4.w);
                const float t = __fadd_rn (z, __shfl_xor_sync (0xffffffffu, z, 16));    // z1 + z2
                m = fmaxf (m, t);                           // == `if (t > m) m = t`: m is never NaN, a NaN t leaves it unchanged
            };
            const int ng = len >> 2;
            // two register sets in turn (no copies): group g + 1 is loaded while group g is on the chain
            float4 va[4], vb[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) va[i] = b4[i * GPC];
#pragma unroll 1
            for (int g = 0; g < ng; g += 2) {
                const int g1 = min (g + 1, GPC - 1), g2 = min (g + 2, GPC - 1);
#pragma unroll
                for (int i = 0; i < 4; ++i) vb[i] = b4[i * GPC + g1];
#pragma unroll
                for (int i = 0; i < 4; ++i) step (va[i]);
                if (g + 1 < ng) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) va[i] = b4[i * GPC + g2];
#pragma unroll
                    for (int i = 0; i < 4; ++i) step (vb[i]);
                }
            }
            for (int j = 4 * ng; j < len; ++j) step (b4[(j & 3) * GPC + (j >> 2)]);       // a block that does not end on a multiple of 4
        }
        if (is_km) {
            // kmeterdsp.cc:80-97: z1 every sample, z2 every 4th; the block's last n%4 samples are ignored
            const int e = min (len, km_n - s0);
            const float4* x4 = reinterpret_cast<const float4*> (&xs[buf][wbase + lane][48]);
            const float om4 = __fmul_rn (4.0f, prm.omega);
            for (int j = 0; j + 4 <= e; j += 4) {
                const float4 v4 = x4[j >> 2];
                const float vv[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float s = __fmul_rn (vv[i], vv[i]);
                    if (kt < s) kt = s;
                    // tolerance mode keeps omega itself (1 - omega would move the 9.72 rad/s corner by 3e-4) and contracts mul + add
                    if (FMA) kz1 = fmaf (prm.omega, __fsub_rn (s, kz1), kz1);
                    else kz1 = __fadd_rn (kz1, __fmul_rn (prm.omega, __fsub_rn (s, kz1)));
                }
                if (FMA) kz2 = fmaf (om4, __fsub_rn (kz1, kz2), kz2);
                else kz2 = __fadd_rn (kz2, __fmul_rn (om4, __fsub_rn (kz1, kz2)));
            }
        }
        if (dr_warp) {
            const float* xr = &xs[buf][drow][48];
            for (int j = 0; j < len; ++j) {
                const float v = xr[j];
                drs = __fadd_rn (drs, __fmul_rn (v, v));
                drp = drp > v ? drp : v;                    // MAX (peak_cur, v) on the RAW sample (:408), NaN-transparent like the macro
                if (s0 + j == wcut) {                        // warp-uniform: the whole warp exchanges, the lanes whose window ends here close
                    const float other = dr.nch == 2 ? __shfl_xor_sync (0xffffffffu, drs, 1) : drs;
                    if (dcut == wcut) {                      // ++scnt > slmt (:410): this lane's 3 s window closes after this sample
                        const bool silent = !((double)drs > dr.silent_thr) && !((double)other > dr.silent_thr);
                        if (dr_live) {
                            dr.emit_valid[dch] = silent ? 0 : 1;
                            if (!silent) { dr.emit_rms[dch] = drs; dr.emit_peak[dch] = drp; }
                        }
                        drs = 0.0f;                          // silent windows keep peak_cur (:293-296)
                        if (!silent) drp = 0.0f;
                    }
                    wcut = __reduce_min_sync (0xffffffffu, dcut > wcut ? dcut : INT_MAX);
                }
            }
        }
        __syncthreads ();                                   // ob / xs[buf] free for reuse
    }
    cp_async_wait<0> ();
    if (dr_live) { dr.rms_sum[dch] = drs; dr.peak_cur[dch] = drp; }

    // ---- end of block --------------------------------------------------------------------
    if (TP) {
        // new history = the 48 samples that precede the next block (left in xs[nchunks&1][.][0..47])
        const int hb = nchunks & 1;
        for (int idx = tid; idx < CH * 48; idx += TPK_THREADS) {
            const int r = idx / 48, j = idx % 48;
            if (c0 + r < n_chan) st.hist[(size_t)(c0 + r) * 48 + j] = xs[hb][r][j];
        }
    }
    if (TP && TPMAX) {
        // process_max (:108-123): m = _res ? 0 : _m; running max; _m = m.  _res, _p, _z1, _z2 untouched.
#pragma unroll
        for (int o = LPR / 2; o; o >>= 1) vmax = fmaxf (vmax, __shfl_xor_sync (0xffffffffu, vmax, o));     // the LPR lanes of row r
        const int ch = c0 + tid / LPR;
        const bool lead = (tid % LPR) == 0 && ch < n_chan;
        float mm = 0.0f;
        if (lead) {
            mm = st.tp_res[ch] ? 0.0f : st.tp_m[ch];
            if (vmax > mm) mm = vmax;
            st.tp_m[ch] = mm;
        }
        if (r128.tpmax) {
            // EBUr128 epilogue: the CH rows span several warps, so their read()s meet in warp 0 (lane = row)
            __shared__ float s_rd[CH];
            if (lead) s_rd[tid / LPR] = mm;
            __syncthreads ();
            if (warp == 0) {
                const float v = lane < CH ? s_rd[lane] : 0.0f;
                const bool own = lane < CH && c0 + lane < n_chan;
                switch (r128.lin ? 0 : r128.nch) {         // the opt-in one-CTA-per-group form: a run-time choice
                case 0: r128_group_hold<0> (r128, st, v, c0 + lane, own); break;
                case 1: r128_group_hold<1> (r128, st, v, c0 + lane, own); break;
                case 4: r128_group_hold<4> (r128, st, v, c0 + lane, own); break;
                default: r128_group_hold<2> (r128, st, v, c0 + lane, own); break;
                }
            }
            // launched with programmatic serialization behind the K-weighting kernel (r128.cu): this grid must not complete
            // before that one has, so that the kernels queued behind it see its results.  Only the LAST CTA to finish waits
            // (griddepcontrol.wait is a no-op in a plain launch): if every CTA waited, the first wave would sit on its SM
            // slots until the slower, latency-bound K-weighting grid ends and the second wave could not start.
            if (tid == 0) {
                const unsigned prev = atomicAdd (st.done_cnt, 1u);
                if (prev == gridDim.x - 1) { *st.done_cnt = 0u; asm volatile ("griddepcontrol.wait;" ::: "memory"); }
            }
        }
    }
    if (is_tp && live) {
        if (filt) st.tp_z2[chs] = __fadd_rn (z, 1e-20f);    // :86-87
        else {
            st.tp_z1[chs] = __fadd_rn (z, 1e-20f);
            m = __fmul_rn (m, prm.g);                       // :89
            if (res) { st.tp_m[chs] = m; st.tp_p[chs] = p; st.tp_res[chs] = 0; }
            else {
                if (m > st.tp_m[chs]) st.tp_m[chs] = m;
                if (p > st.tp_p[chs]) st.tp_p[chs] = p;
            }
        }
    }
    if (is_km && live) {
        if (isnan (kz1)) kz1 = 0;                           // :101-103
        if (isnan (kz2)) kz2 = 0;
        if (!finitef_ (kt)) kt = 0;
        st.km_z1[chs] = __fadd_rn (kz1, 1e-20f);
        st.km_z2[chs] = __fadd_rn (kz2, 1e-20f);
        const float s = __fsqrt_rn (__fmul_rn (2.0f, kz2));
        const float t = __fsqrt_rn (kt);
        if (st.km_flag[chs]) { st.km_rms[chs] = s; st.km_flag[chs] = 0; }
        else if (s > st.km_rms[chs]) st.km_rms[chs] = s;
        float pk = st.km_peak[chs]; int cnt = st.km_cnt[chs];
        if (t >= pk) { pk = t; cnt = prm.hold; }            // :125-139
        else if (cnt > 0) cnt -= nfram;
        else { pk = __fmul_rn (pk, prm.fall); pk = __fadd_rn (pk, 1e-10f); }
        st.km_peak[chs] = pk; st.km_cnt[chs] = cnt;
        st.km_fall[chs] = prm.fall; st.km_fpp[chs] = nfram;
    }
}

// ---- process_max as a grid of independent (channel group x time chunk) CTAs ---------------------------------------------
// TruePeakdsp::process_max (truepeakdsp.cc:101-124) keeps no serial state besides the running maximum, and the FIR is
// time-parallel, so one block is cut into [8 channels x 256 samples] items, one CTA each: 4x more CTAs than tpk_kernel<8,256>
// for a 1024-frame block (8192 for 16384 channels: many waves, so the tail of the last one costs little), no chunk loop, no double buffering, one barrier.  A chunk's 48-sample prefix comes from
// the input itself (chunk 0: from the bank's history); per-chunk maxima meet in blk_max[] with atomicMax on the float bits
// (all values are >= +0, so unsigned order = float order); the CTA that finishes a channel group last applies
// `m = _res ? 0 : _m; if (v > m) m = v; _m = m` and, in the EBUr128 cycle, the plugin's read() x 2 + coef_to_db + tp_max hold.
// The history of the NEXT block goes to the alternate buffer (the group's chunk-0 CTA may still be reading the current one).
// RAG: a ragged EBUr128 block, row c belongs to instance c / r128.nch, which ran for its first rlen[instance] frames.  The maximum
// excludes positions at or after that length (the FIR is causal: the positions before it never see the unread frames); the CTA
// whose chunk holds the row's end writes the row's next history from xs (its 48-sample prefix covers lengths < 48; length 0: chunk 0
// copies the current history, which the host swap would otherwise lose); the epilogue leaves tp_m, tp_res and the hold of a
// length-0 instance untouched (the plugin did not run).
template <bool IMM, bool FMA, int HOLD, bool RAG = false>
__global__ void __launch_bounds__ (TPK_THREADS)
tpmax_kernel (const float* __restrict__ in, size_t stride, int c_first, int n_chan, int nfram, int nchunks, int aligned, int elide0,
              TpkState st, float* __restrict__ dbg, R128Hold r128, const uint32_t* __restrict__ rlen)
{
    constexpr int CH = 8, TC = 256;
    constexpr int XP = 48 + TC + 4;
    constexpr int GPC = TC / 4, LPR = TPK_THREADS / CH;
    __shared__ __align__ (16) float xs[CH][XP];
    __shared__ float s_rowmax[CH];
    const int tid = threadIdx.x, lane = tid & 31;
    const int grp = blockIdx.x / nchunks, chunk = blockIdx.x - grp * nchunks;
    const int c0 = c_first + grp * CH;
    const int s0 = chunk * TC;
    const int len = min (TC, nfram - s0);

    // 48-sample prefix: the bank's history for chunk 0, the input itself otherwise (s0 - 48 is a 16-byte multiple)
    if (chunk == 0) {
        for (int idx = tid; idx < CH * 48; idx += TPK_THREADS) {
            const int r = idx / 48, j = idx % 48;
            cp_async4 (&xs[r][j], st.hist + (size_t)min (c0 + r, n_chan - 1) * 48 + j, 4);
        }
    } else if (aligned) {
        if (tid < CH * 12) {
            const int r = tid / 12, c4 = (tid % 12) * 4;
            cp_async16 (&xs[r][c4], in + (size_t)min (c0 + r, n_chan - 1) * stride + s0 - 48 + c4, 16);
        }
    } else {
        for (int idx = tid; idx < CH * 48; idx += TPK_THREADS) {
            const int r = idx / 48, j = idx % 48;
            cp_async4 (&xs[r][j], in + (size_t)min (c0 + r, n_chan - 1) * stride + s0 - 48 + j, 4);
        }
    }
    if (aligned) {
#pragma unroll
        for (int idx = tid; idx < CH * GPC; idx += TPK_THREADS) {
            const int r = idx / GPC, c4 = (idx % GPC) * 4;
            const int left = (len - c4) * 4;
            const int nb = left >= 16 ? 16 : (left > 0 ? left : 0);
            cp_async16 (&xs[r][48 + c4], nb ? in + (size_t)min (c0 + r, n_chan - 1) * stride + s0 + c4 : in, nb);
        }
    } else {
        for (int idx = tid; idx < CH * TC; idx += TPK_THREADS) {
            const int r = idx / TC, cc = idx % TC;
            const bool ok = cc < len;
            cp_async4 (&xs[r][48 + cc], ok ? in + (size_t)min (c0 + r, n_chan - 1) * stride + s0 + cc : in, ok ? 4 : 0);
        }
    }
    cp_async_commit ();
    cp_async_wait<0> ();
    __syncthreads ();

    const int r = tid / LPR, ql = tid % LPR;
    // positions of this thread's row that count in this chunk
    const int rl = RAG ? max (0, min (len, (int)rlen[(unsigned)min (c0 + r, n_chan - 1) / (unsigned)r128.nch] - s0)) : len;
    float vmax = 0.0f, vmax2 = 0.0f;                        // vmax2: max (|P| + |Q|) = 2 max (|ph1|, |ph3|), tolerance mode
    {
        float M = 0.0f;
        if (elide0) M = row_absmax<LPR, 12 + GPC> (reinterpret_cast<const float4*> (&xs[r][0]), lane);
        const bool silent_rows = elide0 && __all_sync (0xffffffffu, M == 0.0f);      // every phase of a silent row is +0
        if (silent_rows) {
            if (dbg && (c0 + r) < n_chan)
                for (int q = ql; q < GPC && 4 * q < len; q += LPR) {
                    float4* d = reinterpret_cast<float4*> (dbg + (size_t)(c0 + r) * (4 * B200M_MAX_BLOCK) + 4 * (s0 + 4 * q));
#pragma unroll
                    for (int i = 0; i < 4; ++i) d[i] = make_float4 (0.0f, 0.0f, 0.0f, 0.0f);
                }
        } else
#pragma unroll 1
        for (int q = ql; q < GPC; q += LPR) {
            const bool act = 4 * q < rl;
            bool full0 = !FMA;
            if (!FMA && elide0) {
                const float4 xm = *reinterpret_cast<const float4*> (&xs[r][act ? 4 * q + 24 : 0]);
                full0 = !__all_sync (0xffffffffu, !act || phase0_is_delay (xm, M));
            }
            if (act) {
                float w[52];
                const float4* xr = reinterpret_cast<const float4*> (&xs[r][4 * q]);
#pragma unroll
                for (int i = 0; i < 13; ++i) { const float4 v = xr[i]; w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w; }
#if B200M_TPK_SYM
                if (FMA && !dbg) { fir16_fma_max<IMM> (w, min (4, rl - 4 * q), vmax, vmax2); continue; }      // maxima only (dbg: warp-uniform)
#endif
                float o[16];
                if (FMA) fir16_fma<IMM> (w, o); else fir16<IMM> (w, &xs[r][4 * q], o, full0);
                if (dbg && (c0 + r) < n_chan) {
                    float4* d = reinterpret_cast<float4*> (dbg + (size_t)(c0 + r) * (4 * B200M_MAX_BLOCK) + 4 * (s0 + 4 * q));
#pragma unroll
                    for (int i = 0; i < 4; ++i) d[i] = make_float4 (o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
                }
                // positions beyond len inside the last group come from zero-filled input: exclude them
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if (4 * q + i < rl)
                        vmax = fmaxf (fmaxf (vmax, fmaxf (fabsf (o[4 * i]), fabsf (o[4 * i + 1]))), fmaxf (fabsf (o[4 * i + 2]), fabsf (o[4 * i + 3])));
            }
        }
    }
    vmax = fmaxf (vmax, __fmul_rn (0.5f, vmax2));
#pragma unroll
    for (int o = LPR / 2; o; o >>= 1) vmax = fmaxf (vmax, __shfl_xor_sync (0xffffffffu, vmax, o));
    if (ql == 0) s_rowmax[r] = vmax;

    // history of the next block = the 48 samples that end this one (the last chunk holds them: prefix + chunk >= 48 samples)
    if constexpr (RAG) {
        for (int idx = tid; idx < CH * 48; idx += TPK_THREADS) {
            const int rr = idx / 48, j = idx % 48;
            if (c0 + rr >= n_chan) continue;
            const int L = (int)rlen[(unsigned)(c0 + rr) / (unsigned)r128.nch];
            if (chunk == (L > 0 ? (L - 1) / TC : 0)) st.hist_alt[(size_t)(c0 + rr) * 48 + j] = xs[rr][L - s0 + j];
        }
    }
    else if (chunk == nchunks - 1)
        for (int idx = tid; idx < CH * 48; idx += TPK_THREADS) {
            const int rr = idx / 48, j = idx % 48;
            if (c0 + rr < n_chan) st.hist_alt[(size_t)(c0 + rr) * 48 + j] = xs[rr][len + j];
        }
    __syncthreads ();
    if (tid >= 32) return;                                  // the group / grid book-keeping is warp 0's: one fence per CTA, not one per warp

    const int cc = c0 + lane;
    bool own = lane < CH && cc < n_chan;
    if constexpr (RAG) own = own && rlen[(unsigned)cc / (unsigned)r128.nch] != 0;
    if (own && s_rowmax[lane] > 0.0f) atomicMax (st.blk_max + cc, __float_as_uint (s_rowmax[lane]));
    __threadfence ();                                       // the maxima are visible before this CTA's arrival is
    unsigned prev = 0;
    if (lane == 0) prev = atomicAdd (st.grp_cnt + c0, 1u);
    prev = __shfl_sync (0xffffffffu, prev, 0);
    if (prev == (unsigned)(nchunks - 1)) {                  // last chunk of this channel group to finish
        __threadfence ();
        float mm = 0.0f;
        if (own) {
            const float bm = __uint_as_float (atomicExch (st.blk_max + cc, 0u));
            mm = st.tp_res[cc] ? 0.0f : st.tp_m[cc];          // truepeakdsp.cc:108-123
            if (bm > mm) mm = bm;
            st.tp_m[cc] = mm;
        }
        if (r128.tpmax) r128_group_hold<HOLD> (r128, st, mm, cc, own);
        if (lane == 0) st.grp_cnt[c0] = 0u;
    }
    if (r128.tpmax && lane == 0) {
        // launched with programmatic serialization behind the K-weighting kernel (r128.cu): the grid must not complete before
        // that one has.  Only the LAST CTA waits (a no-op in a plain launch); see tpk_kernel's epilogue.
        const unsigned done = atomicAdd (st.done_cnt, 1u);
        if (done == gridDim.x - 1) { *st.done_cnt = 0u; asm volatile ("griddepcontrol.wait;" ::: "memory"); }
    }
}

// ---- process() as a two-stage pipeline over time slabs ---------------------------------------------------------------------
// TruePeakdsp::process (truepeakdsp.cc:41-99) = a time-parallel FIR followed by non-linear ballistics that are strictly serial in
// time.  Fused in one CTA (tpk_kernel<16,64>) the FIR warps wait through every serial phase.  Here the block is cut into slabs
// (sized so that two slabs of |out| fit the L2: 2 x n_chan x slab x 16 B <= 64 MB) and two kernels alternate on two streams:
//   tpfir_kernel  slab s  : one CTA per [8 channels x 64 samples], writes the four |oversampled| values of every input sample to a
//                           scratch slab (float4 per sample, 64 contiguous bytes per thread) -- chip-filling, issue-bound;
//   tpbal_kernel  slab s-1: one CTA per 16 channels: warp 0 = 16 channels x {z1, z2} ballistics lanes reading the scratch slab
//                           (from L2) through cp.async tiles, warp 1 = K-meter lanes (+ DR-14 sums) reading the input block --
//                           latency-bound on its serial chain, runs UNDER the next slab's FIR kernel.
// The per-sample operations and their order are those of tpk_kernel (hence of the reference): results are bit-identical in exact
// mode.  Meter state travels between the slabs of a block through st.tmp; block-begin / block-end transformations (clamp, +1e-20,
// m *= g, read latches) are applied by the first / last slab only.
// The |out| stores between the two kernels are traffic the fused kernel does not have, and the stages only pay off if they overlap.
// Opt-in, bit-identical, covered by tests/test_tpk_gpu.py (fixture mode "slabs"); the fused kernel stays the default.
constexpr int TPF_CH = 8, TPF_TC = 256;

// debugging aid of the slab pipeline (B200M_TPK_TIMELINE=1): every thread 0 stamps %globaltimer into [slot] = {min start, max end}
struct TimelineProbe {
    unsigned long long* p;
    B200M_DEV TimelineProbe (unsigned long long* tl, int slot) : p (tl ? tl + 2 * slot : nullptr)
    {
        if (p && threadIdx.x == 0) { unsigned long long t; asm volatile ("mov.u64 %0, %%globaltimer;" : "=l"(t)); atomicMin (p, t); }
    }
    B200M_DEV ~TimelineProbe ()
    {
        if (p && threadIdx.x == 0) { unsigned long long t; asm volatile ("mov.u64 %0, %%globaltimer;" : "=l"(t)); atomicMax (p + 1, t); }
    }
};

template <bool IMM, bool FMA>
__global__ void __launch_bounds__ (TPK_THREADS)
tpfir_kernel (const float* __restrict__ in, size_t stride, int c_first, int n_chan, int nfram, int s_begin, int s_len, int aligned, int elide0,
              TpkState st, float4* __restrict__ scr, int scr_pitch /* samples per channel row of the slab */, float* __restrict__ dbg,
              unsigned long long* __restrict__ tl /* timeline probe: [slot][2] = first CTA start, last CTA end (globaltimer ns); NULL = off */, int tl_slot)
{
    TimelineProbe tlp (tl, tl_slot);
    constexpr int CH = TPF_CH, TC = TPF_TC;
    constexpr int XP = 48 + TC + 4;                           // LPR = 16 lanes per row: any pitch is conflict free
    constexpr int GPC = TC / 4, LPR = TPK_THREADS / CH;       // 64 groups per row, 16 lanes per row: up to four items per thread
    __shared__ __align__ (16) float xs[CH][XP];
    const int tid = threadIdx.x, lane = tid & 31;
    const int nchunks = (s_len + TC - 1) / TC;
    const int grp = blockIdx.x / nchunks, chunk = blockIdx.x - grp * nchunks;
    const int c0 = c_first + grp * CH;
    const int s0 = s_begin + chunk * TC;                      // absolute sample index inside the block
    const int len = min (TC, s_begin + s_len - s0);
    if (s0 == 0) {
        for (int idx = tid; idx < CH * 48; idx += TPK_THREADS) {
            const int r = idx / 48, j = idx % 48;
            cp_async4 (&xs[r][j], st.hist + (size_t)min (c0 + r, n_chan - 1) * 48 + j, 4);
        }
    } else if (aligned) {
        if (tid < CH * 12) {
            const int r = tid / 12, c4 = (tid % 12) * 4;
            cp_async16 (&xs[r][c4], in + (size_t)min (c0 + r, n_chan - 1) * stride + s0 - 48 + c4, 16);
        }
    } else {
        for (int idx = tid; idx < CH * 48; idx += TPK_THREADS) {
            const int r = idx / 48, j = idx % 48;
            cp_async4 (&xs[r][j], in + (size_t)min (c0 + r, n_chan - 1) * stride + s0 - 48 + j, 4);
        }
    }
    if (aligned) {
#pragma unroll
        for (int idx = tid; idx < CH * GPC; idx += TPK_THREADS) {
            const int r = idx / GPC, c4 = (idx % GPC) * 4;
            const int left = (len - c4) * 4;
            const int nb = left >= 16 ? 16 : (left > 0 ? left : 0);
            cp_async16 (&xs[r][48 + c4], nb ? in + (size_t)min (c0 + r, n_chan - 1) * stride + s0 + c4 : in, nb);      // zero fill beyond the chunk's end
        }
    } else {
        for (int idx = tid; idx < CH * TC; idx += TPK_THREADS) {
            const int r = idx / TC, cc = idx % TC;
            const bool ok = cc < len;
            cp_async4 (&xs[r][48 + cc], ok ? in + (size_t)min (c0 + r, n_chan - 1) * stride + s0 + cc : in, ok ? 4 : 0);
        }
    }
    cp_async_commit ();
    cp_async_wait<0> ();
    __syncthreads ();

    const int r = tid / LPR, ql = tid % LPR;
    float M = 0.0f;
    if (elide0) M = row_absmax<LPR, 12 + GPC> (reinterpret_cast<const float4*> (&xs[r][0]), lane);
    const bool silent_rows = elide0 && __all_sync (0xffffffffu, M == 0.0f);
    const bool rowok = (c0 + r) < n_chan;
#pragma unroll 1
    for (int q = ql; q < GPC && 4 * (q - ql) < len; q += LPR) {
        const bool act = 4 * q < len;
        bool full0 = !FMA;
        if (!FMA && elide0 && !silent_rows) {
            const float4 xm = *reinterpret_cast<const float4*> (&xs[r][act ? 4 * q + 24 : 0]);
            full0 = !__all_sync (0xffffffffu, !act || phase0_is_delay (xm, M));
        }
        if (!act) continue;
        float o[16];
        if (silent_rows) {
#pragma unroll
            for (int i = 0; i < 16; ++i) o[i] = 0.0f;
        } else {
            float w[52];
            const float4* xr = reinterpret_cast<const float4*> (&xs[r][4 * q]);
#pragma unroll
            for (int i = 0; i < 13; ++i) { const float4 v = xr[i]; w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w; }
            if (FMA) fir16_fma<IMM> (w, o); else fir16<IMM> (w, &xs[r][4 * q], o, full0);
        }
        if (!rowok) continue;
        if (dbg) {
            float4* d = reinterpret_cast<float4*> (dbg + (size_t)(c0 + r) * (4 * B200M_MAX_BLOCK) + 4 * (s0 + 4 * q));
#pragma unroll
            for (int i = 0; i < 4; ++i) d[i] = make_float4 (o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
        }
        // |out| of input samples s0 + 4q .. + 3 (positions beyond the block's end are never read by the ballistics kernel)
        float4* d = scr + (size_t)(c0 + r - c_first) * scr_pitch + (s0 - s_begin) + 4 * q;
#pragma unroll
        for (int i = 0; i < 4; ++i) d[i] = make_float4 (fabsf (o[4 * i]), fabsf (o[4 * i + 1]), fabsf (o[4 * i + 2]), fabsf (o[4 * i + 3]));
    }
    // history of the next block = the 48 samples that end this one
    if (s0 + len == nfram)
        for (int idx = tid; idx < CH * 48; idx += TPK_THREADS) {
            const int rr = idx / 48, j = idx % 48;
            if (c0 + rr < n_chan) st.hist_alt[(size_t)(c0 + rr) * 48 + j] = xs[rr][len + j];
        }
}

// samples per scratch tile: 16 channels x 16 samples x 16 B = 4 KB.  Small on purpose: with three stages a CTA holds 17 KB of shared
// memory, so that the ballistics CTAs an SM gets (1024 CTAs for 16384 channels) leave room for the FIR kernel's CTAs of the next slab --
// with 32-sample tiles (32 KB per CTA) whichever kernel was placed first kept the other one off the SM and the two stages ran serially
constexpr int TPB_TILE = 16;
constexpr int TPB_PITCH = 4 * TPB_TILE + 4;                   // floats per channel row: = 4 mod 32
constexpr int TPB_STAGES = 3;

template <bool KM, bool DR>
__global__ void __launch_bounds__ (64, 24)                   // <= 42 registers: seven of these CTAs must leave the register file to the FIR kernel's
tpbal_kernel (const float4* __restrict__ scr, int scr_pitch, const float* __restrict__ in, size_t stride, int c_first, int n_chan, int nch_total, int nfram,
              int s_begin, int s_len, int first, int last, int aligned, int tp_on, TpkParams prm, TpkState st, TpkDr dr,
              unsigned long long* __restrict__ tl, int tl_slot)
{
    TimelineProbe tlp (tl, tl_slot);
    __shared__ __align__ (16) float tile[TPB_STAGES][16 * TPB_PITCH];       // |out| tiles (warp 0)
    __shared__ __align__ (16) float xin[TPB_STAGES][16 * (TPB_TILE + 4)];   // input tiles (warp 1)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int c0 = c_first + blockIdx.x * 16;
    const int ntiles = (s_len + TPB_TILE - 1) / TPB_TILE;
    const size_t N = (size_t)nch_total;                      // st.tmp is [7][channels of the bank]
    if (warp == 0) {
        if (!tp_on) return;
        // ---- true-peak ballistics: lane = filter * 16 + channel (truepeakdsp.cc:52-99)
        const int tch = lane & 15, filt = lane >> 4;
        const int ch = min (c0 + tch, n_chan - 1);
        const bool live = (c0 + tch) < n_chan;
        float z, m, p; int res = 0;
        const float wf = filt ? prm.w2 : prm.w1;
        if (first) {
            res = st.tp_res[ch];
            m = res ? 0.0f : st.tp_m[ch];
            p = res ? 0.0f : st.tp_p[ch];
            const float a = filt ? st.tp_z2[ch] : st.tp_z1[ch];
            z = a > 20 ? 20 : (a < 0 ? 0 : a);
        } else {
            z = st.tmp[(size_t)(filt ? 1 : 0) * N + ch]; m = st.tmp[2 * N + ch]; p = st.tmp[3 * N + ch];
        }
        auto issue = [&] (int t) {
            if (t < ntiles) {
                float* dst = tile[t % TPB_STAGES];
                const int t0 = t * TPB_TILE;
                // 16 rows x TPB_TILE float4 pieces of 16 bytes: lane l takes pieces l, l + 32, ...
#pragma unroll
                for (int i = 0; i < 16 * TPB_TILE / 32; ++i) {
                    const int pc = i * 32 + lane, row = pc / TPB_TILE, col = pc % TPB_TILE;
                    const int chr = min (c0 + row, n_chan - 1) - c_first;
                    const bool ok = (t0 + col) < s_len;
                    cp_async16 (dst + row * TPB_PITCH + 4 * col, ok ? (const void*)(scr + (size_t)chr * scr_pitch + t0 + col) : (const void*)scr, ok ? 16 : 0);
                }
            }
            cp_async_commit ();
        };
#pragma unroll
        for (int t = 0; t < TPB_STAGES - 1; ++t) issue (t);
        for (int t = 0; t < ntiles; ++t) {
            cp_async_wait<TPB_STAGES - 2> ();
            __syncwarp ();
            const float4* b4 = reinterpret_cast<const float4*> (tile[t % TPB_STAGES] + tch * TPB_PITCH);
            const int len = min (TPB_TILE, s_len - t * TPB_TILE);
            float4 nxt = b4[0];
#pragma unroll 4
            for (int j = 0; j < len; ++j) {
                const float4 v4 = nxt;
                nxt = b4[min (j + 1, TPB_TILE - 1)];               // the chain below is ~70 cycles per sample: keep the load off it
                z = __fmul_rn (z, prm.w3);
                const float vv[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    // `if (v > z) z += w (v - z)` without the predicate on the dependency chain: for v <= z (or a NaN v) the increment is
                    // w * max (v - z, 0) = +0 and z + 0 = z exactly (z >= +0 always), otherwise the very same three operations
                    const float v = vv[i];
                    z = __fadd_rn (z, __fmul_rn (wf, fmaxf (__fsub_rn (v, z), 0.0f)));
                    p = fmaxf (p, v);
                }
                const float tt = __fadd_rn (z, __shfl_xor_sync (0xffffffffu, z, 16));
                if (tt > m) m = tt;
            }
            __syncwarp ();
            issue (t + TPB_STAGES - 1);
        }
        cp_async_wait<0> ();
        if (live) {
            if (last) {
                if (first == 0) res = st.tp_res[ch];
                if (filt) st.tp_z2[ch] = __fadd_rn (z, 1e-20f);
                else {
                    st.tp_z1[ch] = __fadd_rn (z, 1e-20f);
                    m = __fmul_rn (m, prm.g);
                    if (res) { st.tp_m[ch] = m; st.tp_p[ch] = p; st.tp_res[ch] = 0; }
                    else {
                        if (m > st.tp_m[ch]) st.tp_m[ch] = m;
                        if (p > st.tp_p[ch]) st.tp_p[ch] = p;
                    }
                }
            } else {
                st.tmp[(size_t)(filt ? 1 : 0) * N + ch] = z;
                if (!filt) { st.tmp[2 * N + ch] = m; st.tmp[3 * N + ch] = p; }
            }
        }
    } else {
        if (!KM) return;
        // ---- warp 1: K-meter on lanes 0..15 (kmeterdsp.cc:74-139), DR-14 window sums on lanes 16..31 (src/dr14.c:401-416)
        const int kch = lane & 15;
        const int ch = min (c0 + kch, n_chan - 1);
        const bool live = (c0 + kch) < n_chan;
        const bool is_km = lane < 16;
        const bool is_dr = DR && dr.rms_sum != nullptr && lane >= 16;
        float kz1 = 0, kz2 = 0, kt = 0, drs = 0, drp = 0;
        // window end of this lane's instance in the block (lanes k and k + 16 share a channel), and the warp's first one at or after
        // this launch's slab: the warp reaches it together, so the silence test's partner exchange is a convergent shuffle
        const int dcut = DR && dr.rms_sum != nullptr ? tpk_dr_cut (dr, ch / dr.nch, nfram) : -1;
        int wcut = DR && dr.rms_sum != nullptr ? __reduce_min_sync (0xffffffffu, dcut >= s_begin ? dcut : INT_MAX) : INT_MAX;
        if (is_km) {
            if (first) {
                const float a = st.km_z1[ch], b = st.km_z2[ch];
                kz1 = a > 50 ? 50 : (a < 0 ? 0 : a);
                kz2 = b > 50 ? 50 : (b < 0 ? 0 : b);
            } else { kz1 = st.tmp[4 * N + ch]; kz2 = st.tmp[5 * N + ch]; kt = st.tmp[6 * N + ch]; }
        }
        if (is_dr) { drs = dr.rms_sum[ch]; drp = dr.peak_cur[ch]; }
        const int km_n = (nfram / 4) * 4;
        constexpr int XPI = TPB_TILE + 4;
        auto issue = [&] (int t) {
            if (t < ntiles) {
                float* dst = xin[t % TPB_STAGES];
                const int t0 = s_begin + t * TPB_TILE;
                if (aligned) {
                    // 16 rows x TPB_TILE / 4 pieces of 16 bytes
#pragma unroll
                    for (int i = 0; i < 16 * (TPB_TILE / 4) / 32; ++i) {
                        const int pc = i * 32 + lane, row = pc / (TPB_TILE / 4), c4 = (pc % (TPB_TILE / 4)) * 4;
                        const int left = (s_begin + s_len - (t0 + c4)) * 4;
                        const int nb = left >= 16 ? 16 : (left > 0 ? left : 0);
                        cp_async16 (dst + row * XPI + c4, nb ? in + (size_t)min (c0 + row, n_chan - 1) * stride + t0 + c4 : in, nb);
                    }
                } else {
                    for (int pc = lane; pc < 16 * TPB_TILE; pc += 32) {
                        const int row = pc / TPB_TILE, col = pc % TPB_TILE;
                        const bool ok = (t0 + col) < s_begin + s_len;
                        cp_async4 (dst + row * XPI + col, ok ? in + (size_t)min (c0 + row, n_chan - 1) * stride + t0 + col : in, ok ? 4 : 0);
                    }
                }
            }
            cp_async_commit ();
        };
#pragma unroll
        for (int t = 0; t < TPB_STAGES - 1; ++t) issue (t);
        const float om4 = __fmul_rn (4.0f, prm.omega);
        for (int t = 0; t < ntiles; ++t) {
            cp_async_wait<TPB_STAGES - 2> ();
            __syncwarp ();
            const float* xr = xin[t % TPB_STAGES] + kch * XPI;
            const int a0 = s_begin + t * TPB_TILE;                     // absolute index of the tile's first sample (a multiple of 4)
            const int len = min (TPB_TILE, s_begin + s_len - a0);
            if (is_km) {
                const int e = min (len, km_n - a0);
                for (int j = 0; j + 4 <= e; j += 4) {
                    const float4 v4 = *reinterpret_cast<const float4*> (xr + j);
                    const float vv[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float sq = __fmul_rn (vv[i], vv[i]);
                        if (kt < sq) kt = sq;
                        kz1 = __fadd_rn (kz1, __fmul_rn (prm.omega, __fsub_rn (sq, kz1)));
                    }
                    kz2 = __fadd_rn (kz2, __fmul_rn (om4, __fsub_rn (kz1, kz2)));
                }
            }
            if (DR && dr.rms_sum != nullptr) {
                for (int j = 0; j < len; ++j) {
                    const float v = xr[j];
                    if (is_dr) { drs = __fadd_rn (drs, __fmul_rn (v, v)); drp = drp > v ? drp : v; }
                    if (a0 + j == wcut) {                           // warp-uniform: both half warps exchange, the lanes whose window ends here close
                        const float other = dr.nch == 2 ? __shfl_xor_sync (0xffffffffu, drs, 1) : drs;
                        if (dcut == wcut) {
                            const bool silent = !((double)drs > dr.silent_thr) && !((double)other > dr.silent_thr);
                            if (is_dr && live) {
                                dr.emit_valid[ch] = silent ? 0 : 1;
                                if (!silent) { dr.emit_rms[ch] = drs; dr.emit_peak[ch] = drp; }
                            }
                            if (is_dr) { drs = 0.0f; if (!silent) drp = 0.0f; }
                        }
                        wcut = __reduce_min_sync (0xffffffffu, dcut > wcut ? dcut : INT_MAX);
                    }
                }
            }
            __syncwarp ();
            issue (t + TPB_STAGES - 1);
        }
        cp_async_wait<0> ();
        if (is_dr && live) { dr.rms_sum[ch] = drs; dr.peak_cur[ch] = drp; }
        if (is_km && live) {
            if (last) {
                if (isnan (kz1)) kz1 = 0;
                if (isnan (kz2)) kz2 = 0;
                if (!finitef_ (kt)) kt = 0;
                st.km_z1[ch] = __fadd_rn (kz1, 1e-20f);
                st.km_z2[ch] = __fadd_rn (kz2, 1e-20f);
                const float sr = __fsqrt_rn (__fmul_rn (2.0f, kz2));
                const float tr = __fsqrt_rn (kt);
                if (st.km_flag[ch]) { st.km_rms[ch] = sr; st.km_flag[ch] = 0; }
                else if (sr > st.km_rms[ch]) st.km_rms[ch] = sr;
                float pk = st.km_peak[ch]; int cnt = st.km_cnt[ch];
                if (tr >= pk) { pk = tr; cnt = prm.hold; }
                else if (cnt > 0) cnt -= nfram;
                else { pk = __fmul_rn (pk, prm.fall); pk = __fadd_rn (pk, 1e-10f); }
                st.km_peak[ch] = pk; st.km_cnt[ch] = cnt;
                st.km_fall[ch] = prm.fall; st.km_fpp[ch] = nfram;
            } else { st.tmp[4 * N + ch] = kz1; st.tmp[5 * N + ch] = kz2; st.tmp[6 * N + ch] = kt; }
        }
    }
}

// ---- process(): the FIR warps and the serial warp of a CTA decoupled ----------------------------------------------------------
// In the fused tpk_kernel<16,64> three of a CTA's four warps wait at the barrier that ends the serial phase while the ballistics warp
// works through its ~21 instructions per input sample, each of which has to win the scheduler against the FIR warps of the other
// resident CTAs.  So the serial work is a fourth ROLE here, as heavy as a FIR warp's share, and never waited for:
//   * three FIR warps (96 threads = 16 rows x 6 groups of 4 samples: one group per thread and 24-sample chunk) produce |out| tiles
//     into a two-deep ring and never wait for the serial warp unless it falls two chunks behind;
//   * one serial warp (lane = filter * 16 + channel, as in the fused kernel) consumes the tiles; it also runs the K-meter: in
//     tolerance mode its four steps per group are folded into one affine step from partial sums the FIR threads compute from their
//     register window (z1 <- z1 - c4 z1 + S); in exact mode it walks the raw samples of the chunk in the input window with the
//     reference's sequential roundings, and the FIR is fir16 with its phase-0 guard evaluated on the thread's own 52-sample window;
//   * the serial warp is warp (blockIdx & 3), so that every SM sub-partition gets the same mix of roles;
//   * the input tile is a sliding window (history + four chunk slots in one row, the 48-sample prefix copied once per lap) instead of
//     two buffers with a prefix copy per chunk; chunk c + 1 is loaded (cp.async, one 16-byte piece per thread) under chunk c's FIR.
//   * the peak-sample reading p is a plain maximum, so the FIR thread reduces its 16 values and the serial warp takes one per group.
// Per CTA and chunk: FIR warps 3 x ~600 warp instructions, serial warp ~24 x 19 = 460.  128 threads, 64 registers, 26 KB of shared
// memory: seven CTAs per SM as before (1024 CTAs for 16384 channels = 0.99 waves).
// Results are bit-identical to the fused kernel (and, in exact mode, to the reference).  The decoupling matters most for small banks,
// where a CTA's own critical path counts: the LV2 facade's batched hubs and the strong-scaling shards run at those sizes.
// Used for banks without the debug tap and without DR-14 accumulation; those run the fused kernel.
constexpr int TPD_CH = 16, TPD_TC = 24, TPD_NSLOT = 4, TPD_FIR = 96;
constexpr int TPD_XL = 48 + TPD_NSLOT * TPD_TC + 8;          // 152 floats = 24 mod 32: the 6 + 2 lanes of a quarter warp (two rows) hit 32 different banks
constexpr int TPD_GPC = TPD_TC / 4;
constexpr int TPD_OP = 4 * TPD_TC + 4;                        // = 4 mod 32: the serial warp's 16 rows read conflict-free
// barrier ids must be immediates: with an id in a register ptxas reserves all 16 named barriers for the CTA, and the SM's barrier
// pool then holds four CTAs instead of seven
template <int ID, int N> B200M_DEV void bar_sync_i () { asm volatile ("bar.sync %0, %1;" :: "n"(ID), "n"(N) : "memory"); }
template <int ID, int N> B200M_DEV void bar_arrive_i () { asm volatile ("bar.arrive %0, %1;" :: "n"(ID), "n"(N) : "memory"); }
template <int ID0, int N> B200M_DEV void bar_sync_2 (int b) { if (b) bar_sync_i<ID0 + 1, N> (); else bar_sync_i<ID0, N> (); }
template <int ID0, int N> B200M_DEV void bar_arrive_2 (int b) { if (b) bar_arrive_i<ID0 + 1, N> (); else bar_arrive_i<ID0, N> (); }

template <bool KM, bool FMA>
__global__ void __launch_bounds__ (TPK_THREADS, 7)
tpdec_kernel (const float* __restrict__ in, size_t stride, int c_first, int n_chan, int nfram, int aligned, int elide0, TpkParams prm, TpkState st)
{
    constexpr int CH = TPD_CH, TC = TPD_TC, GPC = TPD_GPC;
    constexpr int BAR_FIR = 1, BAR_FULL = 2, BAR_EMPTY = 4;
    __shared__ __align__ (16) float xs[CH][TPD_XL];          // [0,48): prefix of slot 0; [48 + 24 k, +24): chunk slot k
    __shared__ __align__ (16) float ob[2][CH][TPD_OP];       // |out| of one chunk: float4 slot i * GPC + q = input sample 4 q + i
    __shared__ __align__ (16) float4 kp[2][CH][GPC];         // per group, from the FIR thread: {K-meter sum kq[i] s_i, max s_i, max |out|, -}
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int c0 = c_first + blockIdx.x * CH;
    const int nchunks = (nfram + TC - 1) / TC;
    if (nchunks == 0) return;
    const int swarp = blockIdx.x & 3;
    const int km_n = (nfram / 4) * 4;                         // "n /= 4" drops n mod 4 samples (kmeterdsp.cc:79)

    if (warp != swarp) {
        // ------------------------------------------------------------------ FIR role
        const int ftid = (warp - (warp > swarp ? 1 : 0)) * 32 + lane;          // 0..95
        const int r = ftid / GPC, q = ftid - GPC * r;
        const float* src = in + (size_t)min (c0 + r, n_chan - 1) * stride;
        auto load_chunk = [&] (int c) {
            const int sa = c * TC + 4 * q;                     // first sample of this thread's piece
            float* dst = &xs[r][48 + (c & (TPD_NSLOT - 1)) * TC + 4 * q];
            if (aligned) {
                const int left = (nfram - sa) * 4;
                const int nb = left >= 16 ? 16 : (left > 0 ? left : 0);
                cp_async16 (dst, nb ? src + sa : in, nb);      // zero fill beyond the block's end
            } else {
#pragma unroll
                for (int i = 0; i < 4; ++i) { const bool ok = sa + i < nfram; cp_async4 (dst + i, ok ? src + sa + i : in, ok ? 4 : 0); }
            }
        };
        for (int idx = ftid; idx < CH * 12; idx += TPD_FIR) {
            const int rr = idx / 12, pc = idx - 12 * rr;
            cp_async16 (&xs[rr][4 * pc], st.hist + (size_t)min (c0 + rr, n_chan - 1) * 48 + 4 * pc, 16);
        }
        load_chunk (0);
        cp_async_commit ();
        for (int c = 0; c < nchunks; ++c) {
            const int slot = c & (TPD_NSLOT - 1), b = c & 1;
            const int s0 = c * TC, len = min (TC, nfram - s0);
            cp_async_wait<0> ();
            bar_sync_i<BAR_FIR, TPD_FIR> ();                    // chunk c is in its slot; every FIR thread is done with chunk c - 1
            if (c + 1 < nchunks) {
                if (slot == TPD_NSLOT - 1)                     // next chunk starts a lap: its prefix = the last 48 samples = slots 2 and 3
                    for (int idx = ftid; idx < CH * 12; idx += TPD_FIR) {
                        const int rr = idx / 12, pc = idx - 12 * rr;
                        *reinterpret_cast<float4*> (&xs[rr][4 * pc]) = *reinterpret_cast<const float4*> (&xs[rr][TPD_NSLOT * TC + 4 * pc]);
                    }
                load_chunk (c + 1);
            }
            cp_async_commit ();
            const bool act = 4 * q < len;
            float o[16]; float4 kpv = make_float4 (0.0f, 0.0f, 0.0f, 0.0f);
            {
                // every thread evaluates its group (beyond the block's end the window is zero-filled): the exact mode's votes below need
                // the whole warp, and only the last chunk of a block has idle groups
                float w[52];
                const float* xw = &xs[r][slot * TC + 4 * q];
                const float4* xr = reinterpret_cast<const float4*> (xw);
#pragma unroll
                for (int i = 0; i < 13; ++i) { const float4 v = xr[i]; w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w; }
                if (FMA) {
                    if (KM) {
                        const float q0 = __fmul_rn (w[48], w[48]), q1 = __fmul_rn (w[49], w[49]), q2 = __fmul_rn (w[50], w[50]), q3 = __fmul_rn (w[51], w[51]);
                        kpv.x = fmaf (prm.kq[3], q3, fmaf (prm.kq[2], q2, fmaf (prm.kq[1], q1, __fmul_rn (prm.kq[0], q0))));
                        kpv.y = fmax3 (fmax3 (q0, q1, q2), q3, 0.0f);
                    }
                    fir16_fma<true> (w, o);
                } else {
                    // exact mode: the reference's unfused sequence (fir16).  Its phase-0 guard and the digital-silence shortcut take the
                    // maximum of |x| over this thread's own 52-sample window (the fused kernel uses the whole row: any superset of the
                    // taps is valid, a tighter one elides more often); both decisions are warp votes, so no branch diverges
                    bool full0 = true, silent = false;
                    if (elide0) {
                        float M = max3_abs_nan (w[0], w[1], w[2]);
#pragma unroll
                        for (int i = 3; i + 1 < 52; i += 2) M = max3_abs_nan (M, w[i], w[i + 1]);
                        M = max3_abs_nan (M, w[51], 0.0f);
                        silent = __all_sync (0xffffffffu, M == 0.0f);
                        full0 = !__all_sync (0xffffffffu, phase0_is_delay (make_float4 (w[24], w[25], w[26], w[27]), M));
                    }
                    if (silent) {
#pragma unroll
                        for (int i = 0; i < 16; ++i) o[i] = 0.0f;
                    } else fir16<true> (w, xw, o, full0);
                }
                // the group's contribution to the peak-sample reading p (`if (v > p) p = v` over every oversampled value, :71): a maximum,
                // so the FIR thread takes it off the serial warp; positions beyond the block's end (zero-filled input) do not count
                const int nv = min (4, len - 4 * q);
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if (i < nv) kpv.z = fmax3 (kpv.z, max3_abs (o[4 * i], o[4 * i + 1], o[4 * i + 2]), fabsf (o[4 * i + 3]));
            }
            if (c >= 2) bar_sync_2<BAR_EMPTY, TPK_THREADS> (b);      // the serial warp is done with chunk c - 2
            if (act) {
                float4* d = reinterpret_cast<float4*> (&ob[b][r][0]);
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    d[i * GPC + q] = make_float4 (fabsf (o[4 * i]), fabsf (o[4 * i + 1]), fabsf (o[4 * i + 2]), fabsf (o[4 * i + 3]));
                kp[b][r][q] = kpv;
            }
            bar_arrive_2<BAR_FULL, TPK_THREADS> (b);              // arrive releases this thread's tile stores to the warp that syncs on the barrier
        }
        // new history = the 48 samples that end the block: they sit right before the end of the last chunk's data
        {
            const int cl = nchunks - 1, base = (cl & (TPD_NSLOT - 1)) * TC + (nfram - cl * TC);
            for (int idx = ftid; idx < CH * 48; idx += TPD_FIR) {
                const int rr = idx / 48, j = idx - 48 * rr;
                if (c0 + rr < n_chan) st.hist[(size_t)(c0 + rr) * 48 + j] = xs[rr][base + j];
            }
        }
    } else {
        // ------------------------------------------------------------------ serial role: lane = filter * 16 + channel
        const int tch = lane & 15, filt = lane >> 4;
        const int chs = min (c0 + tch, n_chan - 1);
        const bool live = (c0 + tch) < n_chan;
        const int res = st.tp_res[chs];
        float m = res ? 0.0f : st.tp_m[chs];                                  // truepeakdsp.cc:52-55
        float p = res ? 0.0f : st.tp_p[chs];
        float z;
        { const float a = filt ? st.tp_z2[chs] : st.tp_z1[chs]; z = a > 20 ? 20 : (a < 0 ? 0 : a); }
        const float wf = filt ? prm.w2 : prm.w1;
        // z <- max (z, (1 - w) z + w' v) with w' = 1 - fl (1 - w), as in tpk_kernel's tolerance mode
        const float omw = __fsub_rn (1.0f, wf), wq = __fsub_rn (1.0f, omw), omw3 = __fmul_rn (omw, prm.w3);
        float kz1 = 0, kz2 = 0, kt = 0;
        if (KM) {
            const float a = st.km_z1[chs], b = st.km_z2[chs];               // kmeterdsp.cc:74-75
            kz1 = a > 50 ? 50 : (a < 0 ? 0 : a);
            kz2 = b > 50 ? 50 : (b < 0 ? 0 : b);
        }
        const float om4 = __fmul_rn (4.0f, prm.omega), nkc4 = -prm.kc4;
        auto step = [&] (const float4 v4) {
            if (FMA) {
                const float zd = __fmul_rn (z, prm.w3);
                z = fmaxf (zd, fmaf (omw3, z, __fmul_rn (wq, v4.x)));
                z = fmaxf (z, fmaf (omw, z, __fmul_rn (wq, v4.y)));
                z = fmaxf (z, fmaf (omw, z, __fmul_rn (wq, v4.z)));
                z = fmaxf (z, fmaf (omw, z, __fmul_rn (wq, v4.w)));
            } else {                                           // truepeakdsp.cc:57-84, operation for operation
                z = __fmul_rn (z, prm.w3);
                if (v4.x > z) z = __fadd_rn (z, __fmul_rn (wf, __fsub_rn (v4.x, z)));
                if (v4.y > z) z = __fadd_rn (z, __fmul_rn (wf, __fsub_rn (v4.y, z)));
                if (v4.z > z) z = __fadd_rn (z, __fmul_rn (wf, __fsub_rn (v4.z, z)));
                if (v4.w > z) z = __fadd_rn (z, __fmul_rn (wf, __fsub_rn (v4.w, z)));
            }
            m = fmaxf (m, __fadd_rn (z, __shfl_xor_sync (0xffffffffu, z, 16)));       // `if (t > m) m = t`: m is never NaN
        };
        for (int c = 0; c < nchunks; ++c) {
            const int b = c & 1, s0 = c * TC, len = min (TC, nfram - s0);
            bar_sync_2<BAR_FULL, TPK_THREADS> (b);
            const float4* b4 = reinterpret_cast<const float4*> (&ob[b][tch][0]);
            const float4* k4 = &kp[b][tch][0];
            // exact mode: the K-meter walks the raw samples of this chunk in the input window (both half warps carry a copy; the slot is
            // not reloaded before this warp has released the chunk after next, see the FIR role)
            const float4* x4 = reinterpret_cast<const float4*> (&xs[tch][48 + (c & (TPD_NSLOT - 1)) * TC]);
            const int ng = len >> 2;
#pragma unroll 2
            for (int g = 0; g < ng; ++g) {
                const float4 v0 = b4[g], v1 = b4[GPC + g], v2 = b4[2 * GPC + g], v3 = b4[3 * GPC + g];
                const float4 k = k4[g];
                step (v0); step (v1); step (v2); step (v3);
                p = fmaxf (p, k.z);
                if (KM && s0 + 4 * g + 4 <= km_n) {
                    if (FMA) {
                        kz1 = __fadd_rn (kz1, fmaf (nkc4, kz1, k.x));
                        kz2 = fmaf (om4, __fsub_rn (kz1, kz2), kz2);
                        kt = fmaxf (kt, k.y);
                    } else {                                   // kmeterdsp.cc:80-97
                        const float4 xv = x4[g];
                        const float vv[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const float sq = __fmul_rn (vv[i], vv[i]);
                            if (kt < sq) kt = sq;
                            kz1 = __fadd_rn (kz1, __fmul_rn (prm.omega, __fsub_rn (sq, kz1)));
                        }
                        kz2 = __fadd_rn (kz2, __fmul_rn (om4, __fsub_rn (kz1, kz2)));
                    }
                }
            }
            if (4 * ng < len) {                                // a block that does not end on a multiple of 4: the last group is partial
                for (int j = 4 * ng; j < len; ++j) step (b4[(j & 3) * GPC + (j >> 2)]);
                p = fmaxf (p, k4[ng].z);
            }
            if (c + 2 < nchunks) bar_arrive_2<BAR_EMPTY, TPK_THREADS> (b);
        }
        if (live) {
            if (filt) st.tp_z2[chs] = __fadd_rn (z, 1e-20f);    // :86-87
            else {
                st.tp_z1[chs] = __fadd_rn (z, 1e-20f);
                m = __fmul_rn (m, prm.g);                       // :89
                if (res) { st.tp_m[chs] = m; st.tp_p[chs] = p; st.tp_res[chs] = 0; }
                else {
                    if (m > st.tp_m[chs]) st.tp_m[chs] = m;
                    if (p > st.tp_p[chs]) st.tp_p[chs] = p;
                }
                if (KM) {
                    if (isnan (kz1)) kz1 = 0;                   // kmeterdsp.cc:101-103
                    if (isnan (kz2)) kz2 = 0;
                    if (!finitef_ (kt)) kt = 0;
                    st.km_z1[chs] = __fadd_rn (kz1, 1e-20f);
                    st.km_z2[chs] = __fadd_rn (kz2, 1e-20f);
                    const float sr = __fsqrt_rn (__fmul_rn (2.0f, kz2));
                    const float tr = __fsqrt_rn (kt);
                    if (st.km_flag[chs]) { st.km_rms[chs] = sr; st.km_flag[chs] = 0; }
                    else if (sr > st.km_rms[chs]) st.km_rms[chs] = sr;
                    float pk = st.km_peak[chs]; int cnt = st.km_cnt[chs];
                    if (tr >= pk) { pk = tr; cnt = prm.hold; }  // :125-139
                    else if (cnt > 0) cnt -= nfram;
                    else { pk = __fmul_rn (pk, prm.fall); pk = __fadd_rn (pk, 1e-10f); }
                    st.km_peak[chs] = pk; st.km_cnt[chs] = cnt;
                    st.km_fall[chs] = prm.fall; st.km_fpp[chs] = nfram;
                }
            }
        }
    }
}

// ---- process_max in tolerance mode on the tensor cores -----------------------------------------------------------------------
// The three non-trivial phases of the 4x oversampler as a Toeplitz GEMM on Hopper's warpgroup MMA (wgmma, tf32), fp32 accuracy from
// the 3xTF32 split:
//   rows     = 16-sample blocks of one channel: 128 rows = 8 channels x 256 samples = the (group, chunk) item of tpmax_kernel;
//   A[r][k]  = x[16 tb - 48 + k], k < 64 (the block's 16 samples and the 48 before them), split x = hi + lo with hi = the top 11
//              significand bits (what a tf32 operand keeps); A is never stored: each thread loads its wgmma A fragments straight
//              from the input stage in shared memory and splits them in registers;
//   B[k][n]  = h_ph[j + 48 - k] for n = 16 (ph - 1) + j, zero outside the 48 taps (h_ph[d] multiplies x[n - d], see fir16), as
//              [B_hi | B_lo] (96 rows) in shared memory, K-major, no swizzle: 8-row x 16-byte core matrices, K chunks 1536 bytes apart;
//   D        = A_hi [B_hi | B_lo] + A_lo B_hi: two instructions per K step (M = 64, K = 8: N = 96 and N = 48, the second one
//              accumulating into the first 48 columns of the first one's registers), 16 per warpgroup and tile; the epilogue adds
//              columns n and 48 + n.  The lo x lo term (2^-20 relative) is dropped.
// Phase 0 of the table is the input delayed by 24 samples (to 7.7e-16, see phase0_is_delay) and is taken from the A fragments directly.
// Roles (persistent CTAs, one per SM; the stages are chained by mbarriers):
//   warp 8      one thread: the tile's 8 rows x 304 floats by cp.async.bulk onto xfull[s], eight stages ahead of the consumers;
//   warps 0-7   two warpgroups, 64 rows of every tile each: A fragments -> registers -> {hi, lo}, 16 wgmmas, maxima over the row's
//               valid positions, per-channel maximum into shared memory; after a group's last chunk: m = max (m, v)
//               (truepeakdsp.cc:108-123) and the EBUr128 epilogue (read x2, coef_to_db, hold).
// Row r of a warp's 16 (wgmma fragment rows g and g + 8, g = lane / 4) is channel r % 8 of the group and 16-sample block
// 8 wg + 2 (warp % 4) + r / 8: the eight row groups of a fragment load then sit 308 floats (= 20 banks) apart, conflict-free.
// A CTA takes WHOLE channel groups and walks their chunks in order, so a block's maximum never leaves the CTA (tpmax_kernel's
// (group, chunk) item grid needs a __threadfence and two global atomics per item).
// Non-finite input: a NaN or Inf sample makes every output of the (up to four) rows whose window holds it NaN, which the maxima
// ignore like the reference ignores its own NaN outputs; |Inf| itself is still seen through phase 0.
// Needs 16-byte aligned rows and nfram % 4 == 0 (bulk copies) and a bank of at least one 8-channel group per SM; everything else runs
// tpmax_kernel.
constexpr int TCF_XPITCH = 308;                            // floats per channel row of an input stage: 48 + 256 + 4; = 20 mod 32
constexpr int TCF_XSTAGES = 8;
constexpr int TCF_BLBO = 96 * 16;                          // bytes between K chunks of [B_hi | B_lo]
constexpr int TCF_BBYTES = 16 * TCF_BLBO;                  // 24576
constexpr int TCF_SMEM = TCF_BBYTES + TCF_XSTAGES * 8 * TCF_XPITCH * 4 + 256;
constexpr int TCF_THREADS = 288;
constexpr int TCF_CONSUMERS = 256;

B200M_DEV uint32_t tcf_smem_u32 (const void* p) { return (uint32_t)__cvta_generic_to_shared (p); }
B200M_DEV uint64_t tcf_desc (uint32_t saddr, uint32_t lbo, uint32_t sbo)      // K-major, no-swizzle wgmma shared-memory matrix descriptor
{
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}
B200M_DEV void tcf_wait (uint32_t bar, uint32_t parity)
{
    uint32_t ok = 0;
    while (!ok) asm volatile ("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
}
B200M_DEV void tcf_arrive (uint32_t bar) { asm volatile ("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory"); }
B200M_DEV void tcf_wgmma_n96 (float (&d)[48], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d)
{
    asm volatile ("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %53, 0;\n\t"
                  "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, {%48, %49, %50, %51}, %52, p, 1, 1;\n\t}\n"
                  : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
                  : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d) : "memory");
}
B200M_DEV void tcf_wgmma_n48 (float (&d)[48], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d)
{
    asm volatile ("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\t"
                  "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, {%24, %25, %26, %27}, %28, p, 1, 1;\n\t}\n"
                  : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
                  : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d) : "memory");
}

// ---- the tile arithmetic, shared by tpmax_tc_kernel and r128_fused_kernel: one thread's part of one 64-row tile, rows g and g + 8
// of its warp, which are two consecutive 16-sample blocks of one channel.  xw = window element t of row g in the input stage.
// A fragment of K step s: a0 = A[g][8s + t], a1 = A[g + 8][8s + t], a2 = A[g][8s + t + 4], a3 = A[g + 8][8s + t + 4]
B200M_DEV void tcf_load (const float* xw, float (&v)[8][4])
{
#pragma unroll
    for (int s = 0; s < 8; ++s) { v[s][0] = xw[8 * s]; v[s][1] = xw[16 + 8 * s]; v[s][2] = xw[8 * s + 4]; v[s][3] = xw[16 + 8 * s + 4]; }
}
// window elements k >= nin[h] (row g: h = 0, row g + 8: h = 1) lie beyond the block's end, where the stage holds stale data: zeroed.
// Returns phase 0's maximum: |window element 24 + j| over the valid output positions j < vj[h].
B200M_DEV float tcf_mask_p0 (float (&v)[8][4], int t, const int (&vj)[2], const int (&nin)[2])
{
    if (nin[1] < 64) {
#pragma unroll
        for (int s = 0; s < 8; ++s)
#pragma unroll
            for (int e = 0; e < 4; ++e)
                if (8 * s + t + 4 * (e >> 1) >= nin[e & 1]) v[s][e] = 0.0f;
    }
    float p0 = 0.0f;
#pragma unroll
    for (int s = 3; s < 5; ++s)
#pragma unroll
        for (int e = 0; e < 4; ++e)
            if (8 * (s - 3) + t + 4 * (e >> 1) < vj[e & 1]) p0 = fmaxf (p0, fabsf (v[s][e]));
    return p0;
}
// x = hi + lo: hi = the top 11 significand bits (what a tf32 operand keeps), lo = the exact remainder
B200M_DEV void tcf_split (const float (&v)[8][4], uint32_t (&ahi)[8][4], uint32_t (&alo)[8][4])
{
#pragma unroll
    for (int s = 0; s < 8; ++s)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const uint32_t hbits = __float_as_uint (v[s][e]) & 0xffffe000u;
            ahi[s][e] = hbits; alo[s][e] = __float_as_uint (__fsub_rn (v[s][e], __uint_as_float (hbits)));
        }
}
// the tile's 16 wgmmas, committed as one group; the first starts the accumulators with scale-d = 0 (no zeroing moves)
B200M_DEV void tcf_mma (float (&d)[48], const uint32_t (&ahi)[8][4], const uint32_t (&alo)[8][4], uint32_t bb)
{
    asm volatile ("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        const uint64_t db = tcf_desc (bb + 2 * s * TCF_BLBO, TCF_BLBO, 128);
        tcf_wgmma_n96 (d, ahi[s], db, s == 0 ? 0u : 1u);                 // A_hi x [B_hi | B_lo]
        tcf_wgmma_n48 (d, alo[s], db, 1u);                               // A_lo x B_hi
    }
    asm volatile ("wgmma.commit_group.sync.aligned;" ::: "memory");
}
B200M_DEV void tcf_mma_wait () { asm volatile ("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// max (mx, |output|) over the valid positions of rows g and g + 8; accumulator registers: d[4i + e] = (row g, column 8i + 2t + e),
// d[4i + 2 + e] = (row g + 8, same column), an output is column n + column 48 + n
B200M_DEV float tcf_tile_max (const float (&d)[48], int t, const int (&vj)[2], float mx)
{
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int j = 8 * (i & 1) + 2 * t + e;
            if (j < vj[0]) mx = fmaxf (mx, fabsf (__fadd_rn (d[4 * i + e], d[4 * (i + 6) + e])));
            if (j < vj[1]) mx = fmaxf (mx, fabsf (__fadd_rn (d[4 * i + 2 + e], d[4 * (i + 6) + 2 + e])));
        }
    return mx;
}

template <int HOLD>
__global__ void __launch_bounds__ (TCF_THREADS, 1)
tpmax_tc_kernel (const float* __restrict__ in, size_t stride, int c_first, int n_chan, int nfram, int nchunks, const float* __restrict__ bcanon,
                 TpkState st, R128Hold r128)
{
    extern __shared__ __align__ (128) uint8_t tcf_smem[];
    uint8_t* sB = tcf_smem;
    float* xbuf = reinterpret_cast<float*> (tcf_smem + TCF_BBYTES);                                        // [XSTAGES][8][XPITCH]
    uint64_t* bars = reinterpret_cast<uint64_t*> (tcf_smem + TCF_BBYTES + TCF_XSTAGES * 8 * TCF_XPITCH * 4);
    uint64_t* xfull = bars; uint64_t* xempty = bars + TCF_XSTAGES;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // a CTA takes whole channel groups (group blockIdx.x, + gridDim.x, ...) and walks each group's chunks in order: the block's maximum
    // of a channel then never leaves the CTA (no global atomics or fences between the chunks, unlike tpmax_kernel's item grid)
    const int ngroups = (n_chan - c_first + 7) / 8;
    const int n_it = (int)blockIdx.x < ngroups ? ((ngroups - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x) * nchunks : 0;
    __shared__ unsigned s_gmax[8];
    if (tid < 8) s_gmax[tid] = 0u;

    for (int i = tid; i < TCF_BBYTES / 16; i += TCF_THREADS) reinterpret_cast<float4*> (sB)[i] = reinterpret_cast<const float4*> (bcanon)[i];
    if (tid == 0) {
        for (int i = 0; i < TCF_XSTAGES; ++i) {
            asm volatile ("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(tcf_smem_u32 (&xfull[i])));
            asm volatile ("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(tcf_smem_u32 (&xempty[i])), "n"(TCF_CONSUMERS));
        }
        asm volatile ("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    asm volatile ("fence.proxy.async.shared::cta;" ::: "memory");             // B: generic-proxy stores, read by the tensor core (async proxy)
    __syncthreads ();

    if (warp == 8) {
        // ---------------- input loads
        if (lane == 0)
            for (int it = 0; it < n_it; ++it) {
                const int sg = it % TCF_XSTAGES;
                if (it >= TCF_XSTAGES) tcf_wait (tcf_smem_u32 (&xempty[sg]), (uint32_t)((it / TCF_XSTAGES - 1) & 1));
                const int gk = it / nchunks, chunk = it - gk * nchunks;
                const int c0 = c_first + ((int)blockIdx.x + gk * (int)gridDim.x) * 8, s0 = chunk * 256;
                const uint32_t xb = tcf_smem_u32 (xbuf + (size_t)sg * 8 * TCF_XPITCH), bar = tcf_smem_u32 (&xfull[sg]);
                const uint32_t nfl = (uint32_t)min (304, nfram - (s0 - 48));      // floats of every row that lie inside the block (or its history)
                asm volatile ("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(8u * nfl * 4u) : "memory");
                for (int cc = 0; cc < 8; ++cc) {
                    const size_t ch = (size_t)min (c0 + cc, n_chan - 1);
                    const uint32_t dst = xb + (uint32_t)(cc * TCF_XPITCH * 4);
                    if (chunk == 0) {                                              // the 48 samples before the block are the bank's history
                        asm volatile ("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                      :: "r"(dst), "l"(st.hist + ch * 48), "r"(192u), "r"(bar) : "memory");
                        asm volatile ("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                      :: "r"(dst + 192u), "l"(in + ch * stride), "r"((nfl - 48u) * 4u), "r"(bar) : "memory");
                    } else
                        asm volatile ("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                      :: "r"(dst), "l"(in + ch * stride + (s0 - 48)), "r"(nfl * 4u), "r"(bar) : "memory");
                }
            }
    } else {
        // ---------------- consumers: warpgroup wg = warp / 4 computes rows 64 wg .. 64 wg + 63 of every tile
        const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
        const int tb0 = 8 * wg + 2 * (warp & 3);                                // blocks of fragment rows g (tb0) and g + 8 (tb0 + 1); channel g
        const uint32_t bb = tcf_smem_u32 (sB);
        for (int it = 0; it < n_it; ++it) {
            const int gk = it / nchunks, chunk = it - gk * nchunks;
            const int c0 = c_first + ((int)blockIdx.x + gk * (int)gridDim.x) * 8, s0 = chunk * 256;
            const int sg = it % TCF_XSTAGES;
            tcf_wait (tcf_smem_u32 (&xfull[sg]), (uint32_t)((it / TCF_XSTAGES) & 1));
            const float* xt = xbuf + (size_t)sg * 8 * TCF_XPITCH;
            const float* xw = xt + g * TCF_XPITCH + 16 * tb0 + t;
            float v[8][4];
            tcf_load (xw, v);
            if (chunk == nchunks - 1 && tid < 96) {
                // history of the next block = the 48 samples that end this one: stage positions nfram - s0 + j (prefix + chunk >= 48 samples)
                const int rr = tid / 12, k4 = (tid - 12 * rr) * 4;
                if (c0 + rr < n_chan)
                    *reinterpret_cast<float4*> (st.hist_alt + (size_t)(c0 + rr) * 48 + k4) = *reinterpret_cast<const float4*> (xt + rr * TCF_XPITCH + (nfram - s0) + k4);
            }
            tcf_arrive (tcf_smem_u32 (&xempty[sg]));
            int vj[2], nin[2];                                                   // valid output positions; window elements k < nin lie inside the block
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                vj[h] = min (16, max (0, nfram - (s0 + 16 * (tb0 + h))));
                nin[h] = nfram - (s0 - 48) - 16 * (tb0 + h);
            }
            const float p0 = tcf_mask_p0 (v, t, vj, nin);
            uint32_t ahi[8][4], alo[8][4];
            tcf_split (v, ahi, alo);
            float d[48];
            tcf_mma (d, ahi, alo, bb);
            tcf_mma_wait ();
            float mx = tcf_tile_max (d, t, vj, p0);
            mx = fmaxf (mx, __shfl_xor_sync (0xffffffffu, mx, 1));
            mx = fmaxf (mx, __shfl_xor_sync (0xffffffffu, mx, 2));
            if (t == 0 && mx > 0.0f) atomicMax (&s_gmax[g], __float_as_uint (mx));
            if (chunk == nchunks - 1) {
                // the group's block is complete: process_max's m = max (m, v) (truepeakdsp.cc:108-123) and the EBUr128 epilogue
                asm volatile ("bar.sync 1, %0;" :: "n"(TCF_CONSUMERS) : "memory");     // every maximum of the group is in s_gmax
                if (warp == 0) {
                    const int cc = c0 + lane;
                    const bool own = lane < 8 && cc < n_chan;
                    float mm = 0.0f;
                    if (lane < 8) { const float bm = __uint_as_float (s_gmax[lane]); s_gmax[lane] = 0u; mm = bm; }
                    if (own) {
                        const float m0 = st.tp_res[cc] ? 0.0f : st.tp_m[cc];
                        if (!(mm > m0)) mm = m0;
                        st.tp_m[cc] = mm;
                    }
                    if (r128.tpmax) r128_group_hold<HOLD> (r128, st, mm, cc, own);
                }
                asm volatile ("bar.sync 1, %0;" :: "n"(TCF_CONSUMERS) : "memory");     // s_gmax is reset before the next group's maxima arrive
            }
        }
    }
    __syncthreads ();
    if (r128.tpmax && tid == 0) {
        // launched with programmatic serialization behind the K-weighting kernel (r128.cu): see tpmax_kernel
        const unsigned dn = atomicAdd (st.done_cnt, 1u);
        if (dn == gridDim.x - 1) { *st.done_cnt = 0u; asm volatile ("griddepcontrol.wait;" ::: "memory"); }
    }
}

// ---- the EBUr128 cycle's K-weighting and true-peak maximum in one persistent kernel (tolerance mode, device path, r128.cu) --------
// One CTA per slab of 128 channels (64 stereo instances; 120 channels for 3 and 5 channels per instance, see the kernel; slabs
// blockIdx.x, + gridDim.x, ...) walks the block in 64-sample stages
// [128 channels][48 history + 64 new + 4 pad] held in a 3-slot shared-memory ring, so the input is read from HBM once for both jobs.
//   warps 0-7   two FIR warpgroups.  Per stage the slab is 512 rows (128 channels x 4 blocks of 16 samples) = 8 m64 tiles, four per
//               warpgroup, computed by tpmax_tc_kernel's tile arithmetic (tcf_*): every maximum is bit-identical to it.  In tile m,
//               warp w of warpgroup wg takes channel 64 wg + 16 m + 8 (w >> 1) + g in rows g / g + 8 and blocks 2 (w & 1), 2 (w & 1) + 1,
//               so a thread meets the same four channels in every stage and keeps their running maxima in registers until the slab
//               ends.  The two warpgroups take turns on the tensor cores (named barriers 2 and 3): one's 16 wgmmas run while the
//               other loads, splits and reduces.
//   warps 8-11  K-weighting: kw_warp<NCHAN, PHASES> (lane = channel) through FusedStage, so the EBU floats stay bit-exact.
// A slot is refilled by the last of the 12 warps to release it (a shared counter), so no role waits for another to finish reading:
// stages >= 1 by one 2-D TMA box [128 rows x 116 floats] from sample 64 t - 48 (rows and samples outside the block read as zero),
// stage 0 by per-row bulk copies of the 48-sample history and the block's first 68 samples.
// Banks: the row pitch 116 = 20 (mod 32) floats puts the rows g = 0..7 of a fragment load (8 consecutive channels, one column) at
// banks 0 20 8 28 16 4 24 12 (+ t = 0..3): 32 different banks.  An LDS.128 phase of a K-weighting warp (8 lanes = 8 consecutive rows,
// one column) covers the same 8 offsets x 4 consecutive banks: conflict-free as well.
constexpr int R128F_CH = 128, R128F_PITCH = 116, R128F_SLOTS = 3, R128F_WARPS = 12;
constexpr int R128F_STAGE_BYTES = R128F_CH * R128F_PITCH * 4;                    // 59392
constexpr int R128F_SMEM = 128 + TCF_BBYTES + R128F_SLOTS * R128F_STAGE_BYTES + 64 + R128F_CH * 4;
static_assert (EBU_TILE == 64, "a stage is one K1 tile");

struct R128fRing {
    uint8_t* stage; uint32_t full, cnt;          // slot 0; full[3] mbarriers, cnt[3] release counters (shared addresses)
    const CUtensorMap* tmap; const float* in; size_t stride; const float* hist; int nch, nfram, ntiles, nslabs, slab;

    B200M_DEV uint8_t* slot (int j) const { return stage + (j % R128F_SLOTS) * R128F_STAGE_BYTES; }
    B200M_DEV void wait (int j) const { tcf_wait (full + 8 * (j % R128F_SLOTS), (uint32_t)(j / R128F_SLOTS) & 1u); }
    // stage j = tile j % ntiles of this CTA's slab j / ntiles into its slot; called by a whole warp
    B200M_DEV void produce (int j, int lane) const
    {
        const int i = j / ntiles, t = j - i * ntiles;
        if (i >= nslabs) return;
        const int c0 = ((int)blockIdx.x + i * (int)gridDim.x) * slab;
        const uint32_t dst = smem_u32 (slot (j)), bar = full + 8 * (j % R128F_SLOTS);
        if (t == 0) {
            // the 48 samples before the block are the bank's history: per-row bulk copies (a TMA box lands densely)
            const uint32_t nb = (uint32_t)min (68, nfram) * 4u;
            if (lane == 0) asm volatile ("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"((uint32_t)R128F_CH * (192u + nb)) : "memory");
            __syncwarp ();
            asm volatile ("fence.proxy.async.shared::cta;" ::: "memory");
            for (int r = lane; r < R128F_CH; r += 32) {
                const size_t ch = (size_t)min (c0 + r, nch - 1);
                const uint32_t d = dst + (uint32_t)(r * R128F_PITCH * 4);
                asm volatile ("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                              :: "r"(d), "l"(hist + ch * 48), "r"(192u), "r"(bar) : "memory");
                asm volatile ("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                              :: "r"(d + 192u), "l"(in + ch * stride), "r"(nb), "r"(bar) : "memory");
            }
        } else if (lane == 0) {
            asm volatile ("fence.proxy.async.shared::cta;" ::: "memory");
            asm volatile ("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"((uint32_t)R128F_STAGE_BYTES) : "memory");
            asm volatile ("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                          :: "r"(dst), "l"(tmap), "r"(64 * t - 48), "r"(c0), "r"(bar) : "memory");
        }
    }
    // a warp is done reading stage j; the last of the 12 warps refills the slot with stage j + 3
    B200M_DEV void release (int j, int lane) const
    {
        __syncwarp ();
        uint32_t old = 0;
        if (lane == 0) asm volatile ("atom.acq_rel.cta.shared::cta.add.u32 %0, [%1], 1;" : "=r"(old) : "r"(cnt + 4 * (j % R128F_SLOTS)) : "memory");
        old = __shfl_sync (0xffffffffu, old, 0);
        if (old % R128F_WARPS == R128F_WARPS - 1) produce (j + R128F_SLOTS, lane);
    }
};

// kw_warp's staging policy in the fused kernel: tile t of slab i is ring stage j0 + t (j0 = i * ntiles), the lane's row from offset 48
struct FusedStage {
    static constexpr int UNROLL = 4;
    R128fRing ring; int j0, lane, row;             // row: byte offset of the lane's first new sample in a slot
    B200M_DEV void prologue () {}
    B200M_DEV void acquire (int t) { ring.wait (j0 + t); }
    B200M_DEV void release (int t) { ring.release (j0 + t, lane); }
    B200M_DEV void drain () {}
    B200M_DEV const float* rowp (int t) const { return reinterpret_cast<const float*> (ring.slot (j0 + t) + row); }
    B200M_DEV float4 ld4 (int t, int q) const { return reinterpret_cast<const float4*> (rowp (t))[q]; }
    B200M_DEV float4 ld4_dyn (int t, int q) const { return ld4 (t, q); }
    B200M_DEV float ld (int t, int e) const { return rowp (t)[e]; }
};

// NCHAN channels per instance: a slab is 4 K-weighting warps of CPW = (32 / NCHAN) NCHAN channels, whole instances only (128
// channels for 1, 2, 4; 120 for 3, 5).  A 120-channel slab still stages and filters 128 rows (the FIR tiles are fixed); rows 120..127
// belong to the next slab (or lie past the bank's end) and are neither reduced nor written back.
// PHASES: the EBU bank's instances have several fragment phases (kw_warp's per-instance cut policy)
template <int NCHAN, bool PHASES>
__global__ void __launch_bounds__ (R128F_WARPS * 32, 1)
r128_fused_kernel (const __grid_constant__ CUtensorMap tmap, const float* __restrict__ in, size_t stride, int nch, int nfram,
                   const float* __restrict__ bcanon, TpkState st, float* __restrict__ r128_tpmax,
                   EbuCoef cf, EbuChunks ck, float fragm_f, float* __restrict__ zst, float* __restrict__ frpwr, float* __restrict__ fragpw, int n_inst)
{
    constexpr int CPW = (32 / NCHAN) * NCHAN, SLAB = 4 * CPW;
    extern __shared__ uint8_t r128f_smem[];
    uint8_t* sB = r128f_smem + ((128u - (smem_u32 (r128f_smem) & 127u)) & 127u);            // TMA destinations: 128-byte aligned
    uint8_t* stages = sB + TCF_BBYTES;
    uint64_t* full = reinterpret_cast<uint64_t*> (stages + R128F_SLOTS * R128F_STAGE_BYTES);
    unsigned* cnt = reinterpret_cast<unsigned*> (full + 4);
    unsigned* s_gmax = reinterpret_cast<unsigned*> (full + 8);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ntiles = (nfram + EBU_TILE - 1) / EBU_TILE, nslabs = (nch + SLAB - 1) / SLAB;
    R128fRing ring;
    ring.stage = stages; ring.full = smem_u32 (full); ring.cnt = smem_u32 (cnt); ring.tmap = &tmap; ring.in = in; ring.stride = stride;
    ring.hist = st.hist; ring.nch = nch; ring.nfram = nfram; ring.ntiles = ntiles; ring.slab = SLAB;
    ring.nslabs = (nslabs - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

    for (int i = tid; i < TCF_BBYTES / 16; i += R128F_WARPS * 32) reinterpret_cast<float4*> (sB)[i] = reinterpret_cast<const float4*> (bcanon)[i];
    if (tid < R128F_CH) s_gmax[tid] = 0u;
    if (tid < R128F_SLOTS) cnt[tid] = 0u;
    if (tid == 0) {
        for (int s = 0; s < R128F_SLOTS; ++s) asm volatile ("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(ring.full + 8 * s));
        asm volatile ("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    asm volatile ("fence.proxy.async.shared::cta;" ::: "memory");             // B: generic-proxy stores, read by the tensor core (async proxy)
    __syncthreads ();

    if (warp >= 8) {
        // ---------------- K-weighting warpgroup: warp kw = CPW channels of the slab; the first one also fills the ring
        const int kw = warp - 8;
        if (kw == 0)
            for (int j = 0; j < R128F_SLOTS; ++j) ring.produce (j, lane);
        FusedStage sg;
        sg.ring = ring; sg.lane = lane; sg.row = ((CPW * kw + lane) * R128F_PITCH + 48) * 4;
        for (int i = 0; i < ring.nslabs; ++i) {
            const int k = ((int)blockIdx.x + i * (int)gridDim.x) * SLAB + CPW * kw + lane;
            sg.j0 = i * ntiles;
            // rows beyond the bank read as zeros (stage 0: the last channel's) and lanes >= CPW read the next warp's rows: neither stores
            kw_warp<NCHAN, PHASES> (sg, lane, min (k, nch - 1), lane < CPW && k < nch, nch, nfram, cf, ck, fragm_f, zst, frpwr, fragpw, n_inst);
        }
        return;
    }

    // ---------------- FIR warpgroups
    const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t4 = lane & 3, b0 = 2 * (w & 1);
    const int rowc = 64 * wg + 8 * (w >> 1) + g;                              // the thread's channel in tile m: rowc + 16 m
    const uint32_t bb = smem_u32 (sB);
    if (wg == 1) bar_arrive_i<2, 256> ();                                     // warpgroup 0 takes the tensor cores first (barrier 2 + wg: its turn)
    for (int i = 0; i < ring.nslabs; ++i) {
        const int c0 = ((int)blockIdx.x + i * (int)gridDim.x) * SLAB;
        float rm0 = 0.0f, rm1 = 0.0f, rm2 = 0.0f, rm3 = 0.0f;                   // running maxima of channels rowc + 16 m, m = 0..3
        for (int t = 0; t < ntiles; ++t) {
            const int j = i * ntiles + t;
            ring.wait (j);
            const float* xs = reinterpret_cast<const float*> (ring.slot (j));
            int vj[2], nin[2];                                                // valid output positions; window elements k < nin lie inside the block
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                vj[h] = min (16, max (0, nfram - (64 * t + 16 * (b0 + h))));
                nin[h] = nfram + 48 - 64 * t - 16 * (b0 + h);
            }
#pragma unroll 1
            for (int m = 0; m < 4; ++m) {
                float v[8][4];
                tcf_load (xs + (rowc + 16 * m) * R128F_PITCH + 16 * b0 + t4, v);
                if (m == 3) {
                    if (t == ntiles - 1) {
                        // history of the next block = the 48 samples that end this one (stage positions nfram - 64 t + k); a warp copies 16 rows
                        for (int q = lane; q < 16 * 12; q += 32) {
                            const int r = 16 * warp + q / 12, k4 = (q % 12) * 4;
                            if ((SLAB == R128F_CH || r < SLAB) && c0 + r < nch)
                                *reinterpret_cast<float4*> (st.hist_alt + (size_t)(c0 + r) * 48 + k4) = *reinterpret_cast<const float4*> (xs + r * R128F_PITCH + (nfram - 64 * t) + k4);
                        }
                    }
                    ring.release (j, lane);
                }
                const float p0 = tcf_mask_p0 (v, t4, vj, nin);
                uint32_t ahi[8][4], alo[8][4];
                tcf_split (v, ahi, alo);
                float d[48];
                // no branch between the wgmmas and their wait (ptxas would serialise them): barrier ids in registers, a predicated arrive
                const uint32_t pass = wg == 0 || i < ring.nslabs - 1 || t < ntiles - 1 || m < 3;
                asm volatile ("bar.sync %0, 256;" :: "r"(2 + wg) : "memory");
                tcf_mma (d, ahi, alo, bb);
                asm volatile ("{ .reg .pred p; setp.ne.b32 p, %1, 0; @p bar.arrive %0, 256; }" :: "r"(3 - wg), "r"(pass) : "memory");
                tcf_mma_wait ();
                // the four maxima rotate: rm0 is always tile m's channel
                const float mx = tcf_tile_max (d, t4, vj, fmaxf (rm0, p0));
                rm0 = rm1; rm1 = rm2; rm2 = rm3; rm3 = mx;
            }
        }
        // the slab's block is complete: one maximum per channel, then process_max's m = max (m, v) (truepeakdsp.cc:108-123) and the
        // EBUr128 epilogue, as in tpmax_tc_kernel
        const float rm[4] = {rm0, rm1, rm2, rm3};
#pragma unroll
        for (int m = 0; m < 4; ++m) {
            float mx = fmaxf (rm[m], __shfl_xor_sync (0xffffffffu, rm[m], 1));
            mx = fmaxf (mx, __shfl_xor_sync (0xffffffffu, mx, 2));
            if (t4 == 0 && mx > 0.0f) atomicMax (&s_gmax[rowc + 16 * m], __float_as_uint (mx));
        }
        bar_sync_i<1, 256> ();
        if (wg == 0) {
            const int cc = c0 + tid;
            const bool own = (SLAB == R128F_CH || tid < SLAB) && cc < nch;
            float mm = __uint_as_float (s_gmax[tid]);
            if (own) {
                const float m0 = st.tp_res[cc] ? 0.0f : st.tp_m[cc];
                if (!(mm > m0)) mm = m0;
                st.tp_m[cc] = mm;
            }
            // src/ebulv2.cc:227-230,360-367 (see r128_group_hold): read() every meter, coef_to_db of the largest, hold
            if constexpr ((NCHAN & (NCHAN - 1)) != 0) {
                // 3 or 5 channels: an instance may straddle two warps, so the reads meet in s_gmax (warpgroup 0: barrier 4)
                if (own) st.tp_res[cc] = 1;
                s_gmax[tid] = __float_as_uint (mm);
                bar_sync_i<4, 128> ();
                if (own && tid % NCHAN == 0) {
                    float t = mm;
#pragma unroll
                    for (int c = 1; c < NCHAN; ++c) { const float b = __uint_as_float (s_gmax[tid + c]); t = t > b ? t : b; }
                    r128_hold (r128_tpmax + cc / NCHAN, t);
                }
                bar_sync_i<4, 128> ();
                s_gmax[tid] = 0u;
            } else {
                s_gmax[tid] = 0u;
                r128_group_hold<NCHAN> (R128Hold {r128_tpmax, nullptr, NCHAN}, st, mm, cc, own);
            }
        }
        bar_sync_i<1, 256> ();                                                // s_gmax is reset before the next slab's maxima arrive
    }
}

// Tried and dropped (round 1): a warp-specialised pipeline for process() — four FIR warps + a K-meter warp in lock
// step, the ballistics warp one chunk behind on a double-buffered |out| tile with full/empty named barriers.  It was
// bit-exact but slower: 48 KB of shared memory and 80 registers x 192 threads cut residency to 4 CTAs/SM, and three role
// bodies (26 KB FIR + ballistics + K-meter) overflow the instruction cache.

__global__ void tpk_read_kernel (int n_chan, uint32_t flags, TpkState st, b200m_tpk_result* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_chan) return;
    b200m_tpk_result r = out[i];
    if (flags & B200M_TPK_TRUEPEAK) { r.tp_m = st.tp_m[i]; r.tp_p = st.tp_p[i]; st.tp_res[i] = 1; }     // read(m,p) :133-138
    if (flags & B200M_TPK_KMETER)   { r.km_rms = st.km_rms[i]; r.km_peak = st.km_peak[i]; st.km_flag[i] = 1; }  // kmeterdsp.cc:150-155
    out[i] = r;
}

// channel `sel`, every channel (sel = -1), or with a list the channels inst[k] * per .. inst[k] * per + per - 1 for k < n_sel
__global__ void tpk_reset_kernel (int n_chan, int sel, uint32_t flags, TpkState st, const uint32_t* inst, int n_sel, int per)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (inst) { if (i >= n_sel * per) return; i = (int)inst[i / per] * per + i % per; }
    if (i >= n_chan || (sel >= 0 && i != sel)) return;
    if (flags & B200M_TPK_TRUEPEAK) { st.tp_res[i] = 1; st.tp_m[i] = 0; st.tp_p[i] = 0; }                 // :140-145
    if (flags & B200M_TPK_KMETER) { st.km_z1[i] = st.km_z2[i] = st.km_rms[i] = st.km_peak[i] = 0; st.km_cnt[i] = 0; st.km_flag[i] = 0; }
    if (flags & 4u) {                                       // b200m_tpk_clear: a fresh meter -- ballistics state and the oversampler's 48-sample history too
        st.tp_z1[i] = st.tp_z2[i] = 0.0f;
        for (int j = 0; j < 48; ++j) { st.hist[(size_t)i * 48 + j] = 0.0f; st.hist_alt[(size_t)i * 48 + j] = 0.0f; }
    }
}

}  // namespace b200m

using namespace b200m;

// ---------------------------------------------------------------------------- host side
struct b200m_tpk {
    int device; uint32_t n_chan, flags; float fsamp;
    TpkParams prm; float ctab[120];
    TpkState st{}; b200m_tpk_result* d_res = nullptr; float* d_dbg = nullptr;
    int imm = 0;                            // host table == literal table: use the immediate-coefficient kernels
    int elide0 = 0;                         // phase 0 of the table is the unit-tap delay fir16's guard assumes
    int split = 1;                          // process() with true peak as the FIR / ballistics slab pipeline (tpfir_kernel + tpbal_kernel); B200M_TPK_SPLIT=0: fused tpk_kernel<16,64>
    float4* d_scr = nullptr; uint32_t slab = 0;       // two slabs of |out|: [2][n_chan][slab] float4
    unsigned long long* d_tl = nullptr; int tl_next = 0;   // B200M_TPK_TIMELINE=1: [4096][2] globaltimer stamps of the pipeline's launches (managed memory)
    cudaStream_t sb = nullptr; cudaEvent_t ev_fir[2] = {nullptr, nullptr}, ev_bal[2] = {nullptr, nullptr};
    int wide = 0, wide_min = 0;             // process() with 64-channel CTAs: opt-in (B200M_TPK_WIDE=1: banks of >= 64 channels per SM, or =<min channels>)
    int dec = 1;                            // process() runs tpdec_kernel (decoupled roles) unless the debug tap or DR-14 sums are on; B200M_TPK_DEC=0: the fused kernel
    int tc = 1;                             // tolerance-mode process_max of large banks on the tensor cores (tpmax_tc_kernel); B200M_TPK_TC=0: tpmax_kernel
    float* d_btc = nullptr; int n_sm = 0;   // [B_hi | B_lo] in wgmma's K-major layout; SM count (persistent grid)
    int chunked = 1;                        // process_max without K-meter runs as (channel group x time chunk) CTAs (tpmax_kernel); B200M_TPK_CHUNKED=0: one CTA per group
    int fma = 0;                            // B200M_PREC_FMA: tolerance-mode FIR (fir16_fma); needs the literal table (imm)
    TpkDr dr{}; bool dr_on = false;         // DR-14 accumulation of the next process() call (set by dr14.cu)
    cudaStream_t own = nullptr; HostStage stage; bool last_host = false;
};

// zita-resampler table for (fr = 1.0, hl = 24, np = 4); restates Resampler_table's constructor
// (zita-resampler/resampler-table.cc:29-44,52-75) in double precision with the host libm.
static void zita_table (float* tab, unsigned hl, unsigned np, double fr)
{
    for (unsigned j = 0; j <= np; ++j) {
        double t = (double)j / (double)np;
        for (unsigned i = 0; i < hl; ++i) {
            double xs = fabs (t * fr), sc = 1.0;
            if (!(xs < 1e-6)) { xs *= M_PI; sc = sin (xs) / xs; }
            double xw = fabs (t / hl), wn = 0.0;
            if (!(xw >= 1.0)) { xw *= M_PI; wn = 0.384 + 0.500 * cos (xw) + 0.116 * cos (2 * xw); }
            tab[j * hl + (hl - i - 1)] = (float)(fr * sc * wn);
            t += 1;
        }
    }
}

static void tpk_design (float fsamp, TpkParams& prm, float* ctab)
{
    // TruePeakdsp::init (truepeakdsp.cc:148-157): float / float / double-literal, rounded to float
    prm.w1 = 4000.0f / fsamp / 4.0;
    prm.w2 = 17200.0f / fsamp / 4.0;
    prm.w3 = 1.0f - 7.0f / fsamp / 4.0;
    prm.g = 0.502f;
    // Kmeterdsp::init (kmeterdsp.cc:47-54)
    prm.hold = (int)(0.5f * fsamp + 0.5f);
    prm.omega = 9.72f / fsamp;
    prm.fall = 0.0f;
    {
        const double om = (double)prm.omega, a = 1.0 - om;
        prm.kq[0] = (float)(om * a * a * a); prm.kq[1] = (float)(om * a * a); prm.kq[2] = (float)(om * a); prm.kq[3] = (float)om;
        prm.kc4 = (float)(1.0 - a * a * a * a);
    }
    zita_table (ctab, 24, 4, 1.0);                  // setup (fsamp, fsamp * 4.0, 1, 24, 1.0): np = 4, ratio-only
}

namespace b200m {
void tpk_set_dr (b200m_tpk* h, const TpkDr* dr) { h->dr_on = dr != nullptr; if (dr) h->dr = *dr; }
const b200m_tpk_result* tpk_device_results (b200m_tpk* h) { return h->d_res; }
int tpk_reset_inst (b200m_tpk* h, const uint32_t* d_inst, uint32_t n_sel, uint32_t per, bool clear, cudaStream_t st)
{
    const uint32_t flags = clear ? h->flags | 4u : h->flags & B200M_TPK_KMETER, n = d_inst ? n_sel * per : h->n_chan;
    tpk_reset_kernel<<<(n + 127) / 128, 128, 0, st>>> ((int)h->n_chan, -1, flags, h->st, d_inst, (int)n_sel, (int)per);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}
}

static cudaStream_t tpk_stream (b200m_tpk* h, void* stream) { return h->last_host ? h->own : (cudaStream_t)stream; }

// the instantiations of the EBUr128 epilogue's HOLD (r128_group_hold)
template <bool IMM, bool FMA, bool RAG = false> static decltype (&tpmax_kernel<IMM, FMA, 2, RAG>) tpmax_kernel_for (int hold)
{
    return hold == 0 ? tpmax_kernel<IMM, FMA, 0, RAG> : hold == 1 ? tpmax_kernel<IMM, FMA, 1, RAG> : hold == 4 ? tpmax_kernel<IMM, FMA, 4, RAG>
                                                                                                       : tpmax_kernel<IMM, FMA, 2, RAG>;
}
static decltype (&tpmax_tc_kernel<2>) tpmax_tc_kernel_for (int hold)
{
    return hold == 0 ? tpmax_tc_kernel<0> : hold == 1 ? tpmax_tc_kernel<1> : hold == 4 ? tpmax_tc_kernel<4> : tpmax_tc_kernel<2>;
}
static const int R128_HOLDS[4] = {0, 1, 2, 4};

// process()/process_max() of every meter; channel slices [bounds[s], bounds[s+1]) are launched separately, slice s
// after event ready[s] when `ready` is given (see ebu_process_sliced).
// rlen (device, one length per EBUr128 instance, r128.nch channels each): a ragged block of the EBUr128 cycle.  It always runs
// tpmax_kernel, exact or FMA: the tensor-core and fused kernels walk whole 8-channel groups through every chunk of the block with
// no per-row end, so only the chunk-parallel kernel has the per-row mask and the per-row history hand-over.
int tpk_process_sliced (b200m_tpk* h, const float* d_in, size_t stride, uint32_t nfram, uint32_t tp_mode, cudaStream_t st,
                        int nsl, const uint32_t* bounds, cudaEvent_t* ready, R128Hold r128, bool pdl, const void* dr_v, const uint32_t* rlen)
{
    const TpkDr* dr = (const TpkDr*)dr_v;
    const bool tp = h->flags & B200M_TPK_TRUEPEAK, km = h->flags & B200M_TPK_KMETER;
    TpkParams prm = h->prm;
    // Kmeterdsp::process (:65-70): per-period fallback multiplier, a pure function of n
    prm.fall = powf (10.0f, -0.05f * 15.0f * ((float)(int)nfram / h->fsamp));
    const int aligned = ((uintptr_t)d_in % 16 == 0) && (stride % 4 == 0);
    dim3 blk (TPK_THREADS);
    bool swap_hist = false;
    for (int sl = 0; sl < nsl; ++sl) {
        const int cf = (int)bounds[sl], ce = (int)bounds[sl + 1];
        if (ce <= cf) continue;
        if (ready) B200M_CUDA (cudaStreamWaitEvent (st, ready[sl], 0));
        // cudaLaunchKernelEx so that the EBUr128 cycle can attach the programmatic-serialization attribute (pdl): the kernel
        // may then start while the K-weighting kernel launched just before it on `st` is still running (r128.cu)
        TpkDr drp = {};
        if (dr && tp && km && tp_mode == B200M_TP_MODE_PROCESS) drp = *dr;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
        cudaLaunchConfig_t cfg = {};
        cfg.blockDim = blk; cfg.dynamicSmemBytes = 0; cfg.stream = st; cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
#define TPK_GO(CH, TC, TP, MX, KM, DRM) do { cfg.gridDim = dim3 ((ce - cf + CH - 1) / CH); cfg.dynamicSmemBytes = TpkGeom<CH, TC, (TP) && !(MX)>::BYTES; \
            if (h->imm && h->fma) B200M_CUDA (cudaLaunchKernelEx (&cfg, tpk_kernel<CH, TC, TP, MX, KM, true, DRM, true>, d_in, stride, cf, ce, (int)nfram, aligned, h->elide0, prm, h->st, h->d_dbg, r128, drp)); \
            else if (h->imm) B200M_CUDA (cudaLaunchKernelEx (&cfg, tpk_kernel<CH, TC, TP, MX, KM, true, DRM>, d_in, stride, cf, ce, (int)nfram, aligned, h->elide0, prm, h->st, h->d_dbg, r128, drp)); \
            else B200M_CUDA (cudaLaunchKernelEx (&cfg, tpk_kernel<CH, TC, TP, MX, KM, false, DRM>, d_in, stride, cf, ce, (int)nfram, aligned, h->elide0, prm, h->st, h->d_dbg, r128, drp)); } while (0)
        if (rlen) {
            const int nchunks = ((int)nfram + 255) / 256;
            cfg.gridDim = dim3 ((unsigned)(((ce - cf + 7) / 8) * nchunks));
            const int hold = r128_hold_of (r128);
            const auto k = h->imm && h->fma ? tpmax_kernel_for<true, true, true> (hold) : h->imm ? tpmax_kernel_for<true, false, true> (hold)
                                                                                                 : tpmax_kernel_for<false, false, true> (hold);
            B200M_CUDA (cudaLaunchKernelEx (&cfg, k, d_in, stride, cf, ce, (int)nfram, nchunks, aligned, h->elide0, h->st, h->d_dbg, r128, rlen));
            swap_hist = true;
        }
        else if (tp && tp_mode == B200M_TP_MODE_MAX && !km && h->chunked && h->tc && h->fma && h->imm && h->d_btc && aligned && nfram % 4 == 0 && !h->d_dbg
            && (ce - cf + 7) / 8 >= h->n_sm) {
            // tensor-core path: persistent CTAs, each takes whole 8-channel groups (a bank too small to give every SM a group runs tpmax_kernel)
            const int nchunks = ((int)nfram + 255) / 256;
            cfg.blockDim = dim3 (TCF_THREADS); cfg.gridDim = dim3 ((unsigned)std::min ((ce - cf + 7) / 8, h->n_sm)); cfg.dynamicSmemBytes = TCF_SMEM;
            B200M_CUDA (cudaLaunchKernelEx (&cfg, tpmax_tc_kernel_for (r128_hold_of (r128)), d_in, stride, cf, ce, (int)nfram, nchunks, (const float*)h->d_btc, h->st, r128));
            cfg.blockDim = blk;
            swap_hist = true;
        }
        else if (tp && tp_mode == B200M_TP_MODE_MAX && !km && h->chunked) {
            // chunk-parallel process_max (tpmax_kernel): the EBUr128 epilogue's groups need c_first to be a multiple of r128.nch (r128.cu)
            const int nchunks = ((int)nfram + 255) / 256;
            cfg.gridDim = dim3 ((unsigned)(((ce - cf + 7) / 8) * nchunks));
            const int hold = r128_hold_of (r128);
            const auto k = h->imm && h->fma ? tpmax_kernel_for<true, true> (hold) : h->imm ? tpmax_kernel_for<true, false> (hold) : tpmax_kernel_for<false, false> (hold);
            B200M_CUDA (cudaLaunchKernelEx (&cfg, k, d_in, stride, cf, ce, (int)nfram, nchunks, aligned, h->elide0, h->st, h->d_dbg, r128, (const uint32_t*)nullptr));
            swap_hist = true;
        }
        else if (tp && tp_mode == B200M_TP_MODE_MAX) { if (km) TPK_GO (8, 256, true, true, true, false); else TPK_GO (8, 256, true, true, false, false); }
        else if (tp && h->split && h->d_scr) {
            // FIR / ballistics slab pipeline: FIR kernels on `st`, ballistics kernels on the bank's second stream, one slab behind
            const int nslab = ((int)nfram + (int)h->slab - 1) / (int)h->slab;
            const int ngrp = (ce - cf + TPF_CH - 1) / TPF_CH, nb16 = (ce - cf + 15) / 16;
            // the ballistics stream must not start before everything queued on `st` so far (previous block's state, controls)
            for (int sidx = 0; sidx < nslab; ++sidx) {
                const int sb0 = sidx * (int)h->slab, sl_len = std::min ((int)h->slab, (int)nfram - sb0), b = sidx & 1;
                float4* scr = h->d_scr + (size_t)b * h->n_chan * h->slab + (size_t)cf * h->slab;
                if (sidx >= 2) B200M_CUDA (cudaStreamWaitEvent (st, h->ev_bal[b], 0));          // the slab buffer is free again
                const int nch = (sl_len + TPF_TC - 1) / TPF_TC;
                if (h->imm && h->fma) tpfir_kernel<true, true><<<ngrp * nch, blk, 0, st>>> (d_in, stride, cf, ce, (int)nfram, sb0, sl_len, aligned, h->elide0, h->st, scr, (int)h->slab, h->d_dbg, h->d_tl, h->tl_next);
                else if (h->imm) tpfir_kernel<true, false><<<ngrp * nch, blk, 0, st>>> (d_in, stride, cf, ce, (int)nfram, sb0, sl_len, aligned, h->elide0, h->st, scr, (int)h->slab, h->d_dbg, h->d_tl, h->tl_next);
                else tpfir_kernel<false, false><<<ngrp * nch, blk, 0, st>>> (d_in, stride, cf, ce, (int)nfram, sb0, sl_len, aligned, h->elide0, h->st, scr, (int)h->slab, h->d_dbg, h->d_tl, h->tl_next);
                B200M_CUDA (cudaEventRecord (h->ev_fir[b], st));
                B200M_CUDA (cudaStreamWaitEvent (h->sb, h->ev_fir[b], 0));
                const int first = sidx == 0, last = sidx == nslab - 1;
                if (km && drp.rms_sum) tpbal_kernel<true, true><<<nb16, 64, 0, h->sb>>> (scr, (int)h->slab, d_in, stride, cf, ce, (int)h->n_chan, (int)nfram, sb0, sl_len, first, last, aligned, 1, prm, h->st, drp, h->d_tl, h->tl_next + 1);
                else if (km) tpbal_kernel<true, false><<<nb16, 64, 0, h->sb>>> (scr, (int)h->slab, d_in, stride, cf, ce, (int)h->n_chan, (int)nfram, sb0, sl_len, first, last, aligned, 1, prm, h->st, drp, h->d_tl, h->tl_next + 1);
                else tpbal_kernel<false, false><<<nb16, 64, 0, h->sb>>> (scr, (int)h->slab, d_in, stride, cf, ce, (int)h->n_chan, (int)nfram, sb0, sl_len, first, last, aligned, 1, prm, h->st, drp, h->d_tl, h->tl_next + 1);
                B200M_CUDA (cudaEventRecord (h->ev_bal[b], h->sb));
                B200M_LAUNCHED (2);
                if (h->d_tl) h->tl_next = (h->tl_next + 2) % 4096;
            }
            B200M_CUDA (cudaStreamWaitEvent (st, h->ev_bal[(nslab - 1) & 1], 0));              // the caller's stream sees the block complete
            if (nslab >= 2) B200M_CUDA (cudaStreamWaitEvent (st, h->ev_bal[(nslab - 2) & 1], 0));
            swap_hist = true;
            continue;
        }
        else if (tp && h->dec && h->imm && !h->d_dbg && !drp.rms_sum) {
            const unsigned grid = (unsigned)((ce - cf + TPD_CH - 1) / TPD_CH);
            if (h->fma) {
                if (km) tpdec_kernel<true, true><<<grid, blk, 0, st>>> (d_in, stride, cf, ce, (int)nfram, aligned, h->elide0, prm, h->st);
                else tpdec_kernel<false, true><<<grid, blk, 0, st>>> (d_in, stride, cf, ce, (int)nfram, aligned, h->elide0, prm, h->st);
            } else {
                if (km) tpdec_kernel<true, false><<<grid, blk, 0, st>>> (d_in, stride, cf, ce, (int)nfram, aligned, h->elide0, prm, h->st);
                else tpdec_kernel<false, false><<<grid, blk, 0, st>>> (d_in, stride, cf, ce, (int)nfram, aligned, h->elide0, prm, h->st);
            }
        }
        else if (tp && h->wide && (ce - cf) >= h->wide_min) {
            // wide CTAs (64 channels x 32-sample chunks): every warp has ballistics lanes, so none idles through the serial phase
            if (km) { if (drp.rms_sum) TPK_GO (64, 32, true, false, true, true); else TPK_GO (64, 32, true, false, true, false); } else TPK_GO (64, 32, true, false, false, false);
        }
        else if (tp) { if (km) { if (drp.rms_sum) TPK_GO (16, 64, true, false, true, true); else TPK_GO (16, 64, true, false, true, false); } else TPK_GO (16, 64, true, false, false, false); }
        else tpk_kernel<16, 64, false, false, true, false, false><<<(ce - cf + 15) / 16, blk, TpkGeom<16, 64, false>::BYTES, st>>> (d_in, stride, cf, ce, (int)nfram, aligned, h->elide0, prm, h->st, h->d_dbg, r128, drp);
#undef TPK_GO
        B200M_LAUNCHED (1);
    }
    if (swap_hist) { float* t = h->st.hist; h->st.hist = h->st.hist_alt; h->st.hist_alt = t; }     // every slice wrote the alternate buffer
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

static int tpk_process (b200m_tpk* h, const float* d_in, size_t stride, uint32_t nfram, uint32_t tp_mode, cudaStream_t st)
{
    const uint32_t bounds[2] = {0, h->n_chan};
    return tpk_process_sliced (h, d_in, stride, nfram, tp_mode, st, 1, bounds, nullptr, R128Hold {}, false, h->dr_on ? &h->dr : nullptr, nullptr);
}

// ---- the EBUr128 cycle's fused K-weighting + true-peak kernel (r128_fused_kernel), launched by the EBU bank in place of K1 (r128.cu)
// It walks time with one CTA per 128-channel slab, so its cycle costs about the same from a few dozen slabs up to one slab per SM,
// while K1 + tpmax_tc_kernel spread any bank over every SM and scale with it.  Cycle of 1024 frames, median of 3 x 300 cycles on an
// H100 80GB HBM3 (SXM, 700 W power limit): two kernels 51.9 / 77.4 / 84.7 / 89.0 / 101.2 / 129.6 us, fused 81.8 / 82.9 / 83.8 / 82.8 /
// 82.5 / 83.4 us for 2048 / 4096 / 4608 / 5120 / 6144 / 8192 stereo instances.  They tie near 4608 instances: banks of at least 10240
// channels (5120 stereo instances) run fused.
constexpr uint32_t R128F_MIN_CH = 10240;

// the history the next block reads (48 floats per channel): after a block, the buffer its kernels left current
float* tpk_hist (b200m_tpk* h) { return h->st.hist; }

bool tpk_r128_fused_ok (const b200m_tpk* h, const float* d_in, size_t stride, uint32_t nfram)
{
    return (h->flags & B200M_TPK_TRUEPEAK) && !(h->flags & B200M_TPK_KMETER) && h->chunked && h->tc && h->fma && h->imm && h->d_btc && !h->d_dbg
        && (uintptr_t)d_in % 16 == 0 && stride % 4 == 0 && nfram % 4 == 0 && h->n_chan >= R128F_MIN_CH;
}

// r128_fused_kernel<nchan, PHASES> as r128f_kernels[nchan - 1][PHASES]
#define R128F_K(N) {r128_fused_kernel<N, false>, r128_fused_kernel<N, true>}
static const decltype (&r128_fused_kernel<2, false>) r128f_kernels[5][2] = {R128F_K (1), R128F_K (2), R128F_K (3), R128F_K (4), R128F_K (5)};
#undef R128F_K

int tpk_r128_fused (b200m_tpk* h, const EbuK1Args& a, float* r128_tpmax, cudaStream_t st)
{
    if (a.nchans != (int)h->n_chan) return set_err (B200M_E_INVAL, "r128: EBU and true-peak banks disagree on the channel count");
    const int nchan = a.nchans / a.n_inst;
    if (nchan < 1 || nchan > 5 || nchan * a.n_inst != a.nchans) return set_err (B200M_E_INVAL, "r128: %d channels per instance", nchan);
    CUtensorMap tm;
    if (!ebu_tma_map (&tm, a.in, a.stride, h->n_chan, (uint32_t)a.nfram, R128F_PITCH, R128F_CH, false))
        return set_err (B200M_E_CUDA, "r128: the driver rejected the input block's tensor map");
    const int slab = 4 * (32 / nchan) * nchan, nslabs = ((int)h->n_chan + slab - 1) / slab;         // r128_fused_kernel's SLAB
    r128f_kernels[nchan - 1][a.ck.fph ? 1 : 0]<<<std::min (nslabs, h->n_sm), R128F_WARPS * 32, R128F_SMEM, st>>> (
        tm, a.in, a.stride, (int)h->n_chan, a.nfram, h->d_btc, h->st, r128_tpmax, a.cf, a.ck, a.fragm_f, a.zst, a.frpwr, a.fragpw, a.n_inst);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    float* t = h->st.hist; h->st.hist = h->st.hist_alt; h->st.hist_alt = t;          // the kernel wrote the next block's history
    return 0;
}

extern "C" {

int b200m_design_tpk (float fsamp, float w[4], float ctab[120], float km[2])
{
    if (!(fsamp >= 1000.0f)) return set_err (B200M_E_INVAL, "bad argument");
    TpkParams p; float t[120]; tpk_design (fsamp, p, t);
    if (w) { w[0] = p.w1; w[1] = p.w2; w[2] = p.w3; w[3] = p.g; }
    if (ctab) memcpy (ctab, t, sizeof (t));
    if (km) { km[0] = p.omega; km[1] = (float)p.hold; }
    return 0;
}

int b200m_tpk_create (b200m_tpk** out, int device, uint32_t n_chan, float fsamp, uint32_t flags)
{
    if (!out) return set_err (B200M_E_INVAL, "NULL out pointer");
    *out = nullptr;
    if (n_chan == 0 || !(fsamp >= 1000.0f) || !(flags & 3u) || (flags & ~3u)) return set_err (B200M_E_INVAL, "bad n_chan/fsamp/flags");
    if (b200m_device_count () <= 0) return set_err (B200M_E_NODEVICE, "no CUDA device: b200meters has no CPU path");
    DeviceGuard g (device);
    if (!g.ok) return set_err (B200M_E_NODEVICE, "cannot select CUDA device %d", device);
    b200m_tpk* h = new (std::nothrow) b200m_tpk;
    if (!h) return set_err (B200M_E_NOMEM, "host allocation failed");
    h->device = device; h->n_chan = n_chan; h->flags = flags; h->fsamp = fsamp;
    tpk_design (fsamp, h->prm, h->ctab);
    h->imm = memcmp (h->ctab, h_zita_lit, sizeof (h->ctab)) == 0;
    if (const char* v = getenv ("B200M_TPK_IMM")) h->imm = h->imm && atoi (v);
    // the phase-0 guard's bound (see phase0_is_delay) holds for this table: unit tap at [23], the other 46 taps sum to <= 7.71e-16
    {
        double S = 0.0;
        for (int i = 0; i < 24; ++i) S += (i == 23 ? 0.0 : fabs ((double)h->ctab[i])) + fabs ((double)h->ctab[96 + i]);
        h->elide0 = h->ctab[23] == 1.0f && S <= 7.71e-16;
    }
    if (const char* v = getenv ("B200M_TPK_ELIDE0")) h->elide0 = h->elide0 && atoi (v);      // 0: always evaluate phase 0 (tests, worst-case timing)
    if (const char* v = getenv ("B200M_TPK_PRECISION")) h->fma = (strcmp (v, "fma") == 0) && h->imm && h->ctab[23] == 1.0f;
    cudaError_t e = cudaMemcpyToSymbol (c_tp_tab, h->ctab, sizeof (h->ctab));
    // the process_max kernels share SMs with the K-weighting kernel in the EBUr128 cycle: same (maximum) carveout, so that the SM
    // need not be reconfigured between the two
    if (e == cudaSuccess) e = cudaFuncSetAttribute (tpk_kernel<8, 256, true, true, false, true, false, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e == cudaSuccess) e = cudaFuncSetAttribute (tpk_kernel<8, 256, true, true, false, true, false, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e == cudaSuccess) e = cudaFuncSetAttribute (tpk_kernel<8, 256, true, true, false, false, false, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    // seven CTAs x 24 KB per SM: without the hint the driver may pick a carveout that fits four
    if (e == cudaSuccess) e = cudaFuncSetAttribute (tpdec_kernel<true, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e == cudaSuccess) e = cudaFuncSetAttribute (tpdec_kernel<false, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e == cudaSuccess) e = cudaFuncSetAttribute (tpdec_kernel<true, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e == cudaSuccess) e = cudaFuncSetAttribute (tpdec_kernel<false, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    for (const int hold : R128_HOLDS)
        for (const auto k : {tpmax_kernel_for<true, true> (hold), tpmax_kernel_for<true, false> (hold), tpmax_kernel_for<false, false> (hold),
                             tpmax_kernel_for<true, true, true> (hold), tpmax_kernel_for<true, false, true> (hold), tpmax_kernel_for<false, false, true> (hold)})
            if (e == cudaSuccess) e = cudaFuncSetAttribute (k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    auto A = [&] (void** p, size_t bytes) { if (e == cudaSuccess) { e = cudaMalloc (p, bytes); if (e == cudaSuccess) e = cudaMemset (*p, 0, bytes); } };
    const size_t n = n_chan;
    A ((void**)&h->st.hist, n * 48 * sizeof (float));
    A ((void**)&h->st.tp_z1, n * 4); A ((void**)&h->st.tp_z2, n * 4); A ((void**)&h->st.tp_m, n * 4); A ((void**)&h->st.tp_p, n * 4);
    A ((void**)&h->st.tp_res, n * 4);
    A ((void**)&h->st.km_z1, n * 4); A ((void**)&h->st.km_z2, n * 4); A ((void**)&h->st.km_rms, n * 4); A ((void**)&h->st.km_peak, n * 4);
    A ((void**)&h->st.km_fall, n * 4); A ((void**)&h->st.km_cnt, n * 4); A ((void**)&h->st.km_fpp, n * 4); A ((void**)&h->st.km_flag, n * 4);
    A ((void**)&h->d_res, n * sizeof (b200m_tpk_result));
    A ((void**)&h->st.done_cnt, 16);
    A ((void**)&h->st.hist_alt, n * 48 * sizeof (float));
    A ((void**)&h->st.blk_max, n * 4); A ((void**)&h->st.grp_cnt, n * 4);
    if (const char* v = getenv ("B200M_TPK_CHUNKED")) h->chunked = atoi (v) != 0;
    if (const char* v = getenv ("B200M_TPK_TC")) h->tc = atoi (v) != 0;
    if ((flags & B200M_TPK_TRUEPEAK) && h->imm && e == cudaSuccess) {
        // B[k][n] = h_ph[j + 48 - k] for n = 16 (ph - 1) + j: h_ph[d] multiplies x[n - d] (fir16: d >= 24 -> tab[24 ph + 47 - d], else tab[24 (4 - ph) + d]);
        // element (n, k) of the hi part at (k / 4) * 1536 + n * 16 + (k % 4) * 4 bytes, the lo part 48 rows further
        float* hb = new (std::nothrow) float[TCF_BBYTES / 4];
        if (hb) {
            memset (hb, 0, TCF_BBYTES);
            for (int n = 0; n < 48; ++n) for (int k = 0; k < 64; ++k) {
                const int ph = n / 16 + 1, j = n % 16, d = j + 48 - k;
                const float c = (d >= 0 && d <= 47) ? (d >= 24 ? h->ctab[24 * ph + 47 - d] : h->ctab[24 * (4 - ph) + d]) : 0.0f;
                uint32_t u; memcpy (&u, &c, 4); u &= 0xffffe000u; float hi; memcpy (&hi, &u, 4);
                const size_t off = ((size_t)(k / 4) * TCF_BLBO + (size_t)n * 16 + (size_t)(k % 4) * 4) / 4;
                hb[off] = hi; hb[off + 48 * 4] = c - hi;
            }
            e = cudaMalloc ((void**)&h->d_btc, TCF_BBYTES);
            if (e == cudaSuccess) e = cudaMemcpy (h->d_btc, hb, TCF_BBYTES, cudaMemcpyHostToDevice);
            delete[] hb;
        }
        // it shares SMs with the K-weighting kernel in the EBUr128 cycle (106 KB + 104 KB): same (maximum) carveout as that one
        for (const int hold : R128_HOLDS) {
            if (e == cudaSuccess) e = cudaFuncSetAttribute (tpmax_tc_kernel_for (hold), cudaFuncAttributeMaxDynamicSharedMemorySize, TCF_SMEM);
            if (e == cudaSuccess) e = cudaFuncSetAttribute (tpmax_tc_kernel_for (hold), cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        }
        for (const auto& kp : r128f_kernels)
            for (const auto k : kp) if (e == cudaSuccess) e = cudaFuncSetAttribute (k, cudaFuncAttributeMaxDynamicSharedMemorySize, R128F_SMEM);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute (&h->n_sm, cudaDevAttrMultiProcessorCount, device);
    }
    if (const char* v = getenv ("B200M_TPK_DEC")) h->dec = atoi (v) != 0;
    // the slab pipeline is opt-in (B200M_TPK_SPLIT=2; =1: for banks of >= 512 channels): MEASURED slower than the fused kernel, see below
    h->split = 0;
    if (const char* v = getenv ("B200M_TPK_SPLIT")) { const int q = atoi (v); h->split = q >= 2 ? 1 : (q == 1 ? n_chan >= 512 : 0); }
    A ((void**)&h->st.tmp, 7 * n * sizeof (float));
    { const char* v = getenv ("B200M_TPK_STAGGER"); if (v && atoi (v) != 0) A ((void**)&h->st.sm_arr, 256 * sizeof (unsigned)); }      // opt-in: measured no gain
    if ((flags & B200M_TPK_TRUEPEAK) && h->split) {
        // slab length: two slabs of |out| (16 B per sample and channel) within 64 MB, so that the ballistics kernel reads them from L2
        uint32_t slab = 64;
        while (slab < B200M_MAX_BLOCK && (size_t)2 * n * (2 * slab) * 16 <= ((size_t)64 << 20)) slab *= 2;
        if (const char* v = getenv ("B200M_TPK_SLAB")) { const int q = atoi (v); if (q >= 64 && q <= (int)B200M_MAX_BLOCK && q % 64 == 0) slab = (uint32_t)q; }
        h->slab = slab;
        if (const char* v = getenv ("B200M_TPK_TIMELINE")) if (atoi (v) && e == cudaSuccess) {
            e = cudaMallocManaged ((void**)&h->d_tl, 4096 * 2 * sizeof (unsigned long long));
            if (e == cudaSuccess) for (int i = 0; i < 4096; ++i) { h->d_tl[2 * i] = ~0ull; h->d_tl[2 * i + 1] = 0ull; }
        }
        A ((void**)&h->d_scr, (size_t)2 * n * slab * sizeof (float4));
        // the ballistics kernels are latency-bound and small: highest stream priority, so that SM slots freed by retiring FIR CTAs go to
        // them first (at equal priority the FIR grid keeps the register file full and lets one ballistics CTA per SM in at a time)
        int prio_lo = 0, prio_hi = 0;
        if (e == cudaSuccess) e = cudaDeviceGetStreamPriorityRange (&prio_lo, &prio_hi);
        if (e == cudaSuccess) e = cudaStreamCreateWithPriority (&h->sb, cudaStreamNonBlocking, prio_hi);
        for (int i = 0; i < 2; ++i) {
            if (e == cudaSuccess) e = cudaEventCreateWithFlags (&h->ev_fir[i], cudaEventDisableTiming);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags (&h->ev_bal[i], cudaEventDisableTiming);
        }
    }
    if (const char* v = getenv ("B200M_TPK_WIDE")) {
        const int w = atoi (v); h->wide = w != 0;
        if (w > 1) h->wide_min = w;
        else if (e == cudaSuccess) { int nsm = 0; e = cudaDeviceGetAttribute (&nsm, cudaDevAttrMultiProcessorCount, device); h->wide_min = 64 * nsm; }
    }
    // the wide process() kernels need 87 KB of dynamic shared memory
#define TPK_WATTR(KMF, DRF, FMAF) if (e == cudaSuccess) e = cudaFuncSetAttribute (tpk_kernel<64, 32, true, false, KMF, true, DRF, FMAF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TpkGeom<64, 32, true>::BYTES)
    TPK_WATTR (true, true, true); TPK_WATTR (true, true, false); TPK_WATTR (true, false, true); TPK_WATTR (true, false, false); TPK_WATTR (false, false, true); TPK_WATTR (false, false, false);
#undef TPK_WATTR
    if (e == cudaSuccess) e = cudaFuncSetAttribute (tpk_kernel<64, 32, true, false, true, false, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TpkGeom<64, 32, true>::BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute (tpk_kernel<64, 32, true, false, true, false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TpkGeom<64, 32, true>::BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute (tpk_kernel<64, 32, true, false, false, false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TpkGeom<64, 32, true>::BYTES);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags (&h->own, cudaStreamNonBlocking);
    if (e == cudaSuccess) {
        // constructors: TruePeakdsp _res(true) (:29); Kmeterdsp _flag(false), all zero (kmeterdsp.cc:30-40);
        // the 8192-zero pre-roll (:159-168) leaves an all-zero history, which the memset above provides
        tpk_reset_kernel<<<(n_chan + 127) / 128, 128>>> ((int)n_chan, -1, B200M_TPK_TRUEPEAK, h->st, nullptr, 0, 1);
        B200M_LAUNCHED (1);
        e = cudaDeviceSynchronize ();
    }
    if (e != cudaSuccess) { int rc = cuda_fail (e, "tpk_create", __FILE__, __LINE__); b200m_tpk_destroy (h); return rc; }
    *out = h;
    return 0;
}

int b200m_tpk_destroy (b200m_tpk* h)
{
    if (!h) return 0;
    DeviceGuard g (h->device);
    cudaDeviceSynchronize ();
    void* ps[] = {h->st.hist, h->st.tp_z1, h->st.tp_z2, h->st.tp_m, h->st.tp_p, h->st.tp_res, h->st.km_z1, h->st.km_z2, h->st.km_rms,
                  h->st.km_peak, h->st.km_fall, h->st.km_cnt, h->st.km_fpp, h->st.km_flag, h->d_res, h->d_dbg, h->st.done_cnt, h->st.hist_alt, h->st.blk_max, h->st.grp_cnt, h->st.tmp, h->d_scr, h->st.sm_arr, h->d_tl, h->d_btc};
    for (void* p : ps) cudaFree (p);
    if (h->sb) cudaStreamDestroy (h->sb);
    for (int i = 0; i < 2; ++i) { if (h->ev_fir[i]) cudaEventDestroy (h->ev_fir[i]); if (h->ev_bal[i]) cudaEventDestroy (h->ev_bal[i]); }
    h->stage.release ();
    if (h->own) cudaStreamDestroy (h->own);
    delete h;
    return 0;
}

int b200m_tpk_process_device (b200m_tpk* h, const float* d_in, size_t stride, uint32_t nfram, uint32_t tp_mode, void* stream)
{
    if (int rc = check_block_args (h, d_in, stride, nfram)) return rc;
    if (tp_mode > 1) return set_err (B200M_E_INVAL, "bad tp_mode %u", tp_mode);
    DeviceGuard g (h->device);
    h->last_host = false;
    return tpk_process (h, d_in, stride, nfram, tp_mode, (cudaStream_t)stream);
}

int b200m_tpk_process_host (b200m_tpk* h, const float* in, size_t stride, uint32_t nfram, uint32_t tp_mode)
{
    if (int rc = check_block_args (h, in, stride, nfram)) return rc;
    if (tp_mode > 1) return set_err (B200M_E_INVAL, "bad tp_mode %u", tp_mode);
    DeviceGuard g (h->device);
    B200M_ENTER_HOST_PATH (h);
    if (h->stage.ensure (h->n_chan, nfram)) return set_err (B200M_E_NOMEM, "staging buffer allocation failed");
    B200M_CUDA (cudaMemcpy2DAsync (h->stage.d, h->stage.cap * sizeof (float), in, stride * sizeof (float),
                                   (size_t)nfram * sizeof (float), h->n_chan, cudaMemcpyHostToDevice, h->own));
    h->last_host = true;
    return tpk_process (h, h->stage.d, h->stage.cap, nfram, tp_mode, h->own);
}

int b200m_tpk_set_precision (b200m_tpk* h, int mode)
{
    if (!h || (mode != B200M_PREC_EXACT && mode != B200M_PREC_FMA)) return set_err (B200M_E_INVAL, "bad argument");
    if (mode == B200M_PREC_FMA && !(h->imm && h->ctab[23] == 1.0f)) return set_err (B200M_E_UNSUPPORTED, "tolerance mode needs the literal zita table");
    h->fma = mode == B200M_PREC_FMA;                      // takes effect with the next process call
    return 0;
}
int b200m_tpk_precision (const b200m_tpk* h) { return h ? (h->fma ? B200M_PREC_FMA : B200M_PREC_EXACT) : B200M_E_INVAL; }

int b200m_tpk_read_device (b200m_tpk* h, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    DeviceGuard g (h->device);
    tpk_read_kernel<<<(h->n_chan + 255) / 256, 256, 0, tpk_stream (h, stream)>>> ((int)h->n_chan, h->flags, h->st, h->d_res);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

int b200m_tpk_results (b200m_tpk* h, b200m_tpk_result* out, void* stream)
{
    if (!h || !out) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = tpk_stream (h, stream);
    B200M_CUDA (cudaMemcpyAsync (out, h->d_res, h->n_chan * sizeof (b200m_tpk_result), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_tpk_reset (b200m_tpk* h, int32_t chan, void* stream)
{
    if (!h || chan >= (int32_t)h->n_chan) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    tpk_reset_kernel<<<(h->n_chan + 127) / 128, 128, 0, tpk_stream (h, stream)>>> ((int)h->n_chan, chan, h->flags, h->st, nullptr, 0, 1);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

int b200m_tpk_clear (b200m_tpk* h, int32_t chan, void* stream)
{
    // reset() plus what a newly constructed meter has: zero ballistics filters and an all-zero resampler history (the state after
    // TruePeakdsp::init's pre-roll, truepeakdsp.cc:159-168).  For slot reuse in shared banks.
    if (!h || chan >= (int32_t)h->n_chan) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    tpk_reset_kernel<<<(h->n_chan + 127) / 128, 128, 0, tpk_stream (h, stream)>>> ((int)h->n_chan, chan, h->flags | 4u, h->st, nullptr, 0, 1);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

int b200m_tpk_reset_kmeter (b200m_tpk* h, void* stream)
{
    // reset_peaks of the TPnRMS/DR14 plugin resets only its K-meters (src/dr14.c:241-258)
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    DeviceGuard g (h->device);
    tpk_reset_kernel<<<(h->n_chan + 127) / 128, 128, 0, tpk_stream (h, stream)>>> ((int)h->n_chan, -1, h->flags & B200M_TPK_KMETER, h->st, nullptr, 0, 1);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

// ---- snapshot / restore: header + every per-channel state array in TpkState order
namespace {
struct TpkSnapHead { uint32_t magic, n_chan, flags; float fsamp; };
constexpr uint32_t TPK_SNAP_MAGIC = 0x50543031u;              // "TP01"
int tpk_segments (b200m_tpk* h, void** p, size_t* b)
{
    const size_t n = h->n_chan;
    void* ps[] = {h->st.hist, h->st.tp_z1, h->st.tp_z2, h->st.tp_m, h->st.tp_p, h->st.tp_res, h->st.km_z1, h->st.km_z2, h->st.km_rms, h->st.km_peak,
                  h->st.km_fall, h->st.km_cnt, h->st.km_fpp, h->st.km_flag, h->d_res};
    const size_t bs[] = {n * 48 * 4, n * 4, n * 4, n * 4, n * 4, n * 4, n * 4, n * 4, n * 4, n * 4, n * 4, n * 4, n * 4, n * 4, n * sizeof (b200m_tpk_result)};
    for (int i = 0; i < 15; ++i) { p[i] = ps[i]; b[i] = bs[i]; }
    return 15;
}
}

size_t b200m_tpk_snapshot_size (b200m_tpk* h)
{
    if (!h) return 0;
    void* p[15]; size_t b[15]; const int k = tpk_segments (h, p, b);
    size_t t = 16;
    for (int i = 0; i < k; ++i) t += (b[i] + 15) & ~size_t (15);
    return t;
}

int b200m_tpk_snapshot (b200m_tpk* h, void* buf, size_t bytes, void* stream)
{
    if (!h || !buf || bytes < b200m_tpk_snapshot_size (h)) return set_err (B200M_E_INVAL, "bad argument / buffer too small");
    DeviceGuard g (h->device);
    cudaStream_t st = tpk_stream (h, stream);
    const TpkSnapHead hd = {TPK_SNAP_MAGIC, h->n_chan, h->flags, h->fsamp};
    memcpy (buf, &hd, sizeof (hd));
    uint8_t* o = (uint8_t*)buf + 16;
    void* p[15]; size_t b[15]; const int k = tpk_segments (h, p, b);
    for (int i = 0; i < k; ++i) { B200M_CUDA (cudaMemcpyAsync (o, p[i], b[i], cudaMemcpyDeviceToHost, st)); o += (b[i] + 15) & ~size_t (15); }
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_tpk_restore (b200m_tpk* h, const void* buf, size_t bytes, void* stream)
{
    if (!h || !buf || bytes < b200m_tpk_snapshot_size (h)) return set_err (B200M_E_INVAL, "bad argument / buffer too small");
    TpkSnapHead hd; memcpy (&hd, buf, sizeof (hd));
    if (hd.magic != TPK_SNAP_MAGIC || hd.n_chan != h->n_chan || hd.flags != h->flags || hd.fsamp != h->fsamp)
        return set_err (B200M_E_INVAL, "snapshot does not match this bank (channels / meters / sample rate)");
    DeviceGuard g (h->device);
    cudaStream_t st = tpk_stream (h, stream);
    const uint8_t* o = (const uint8_t*)buf + 16;
    void* p[15]; size_t b[15]; const int k = tpk_segments (h, p, b);
    for (int i = 0; i < k; ++i) { B200M_CUDA (cudaMemcpyAsync (p[i], o, b[i], cudaMemcpyHostToDevice, st)); o += (b[i] + 15) & ~size_t (15); }
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_tpk_coeffs (const b200m_tpk* h, float w[4], float ctab[120], float km[2])
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    if (w) { w[0] = h->prm.w1; w[1] = h->prm.w2; w[2] = h->prm.w3; w[3] = h->prm.g; }
    if (ctab) memcpy (ctab, h->ctab, sizeof (h->ctab));
    if (km) { km[0] = h->prm.omega; km[1] = (float)h->prm.hold; }
    return 0;
}

int b200m_tpk_state (b200m_tpk* h, float* tp_m, float* tp_p, float* tp_z1, float* tp_z2, int32_t* tp_res, float* km8, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    DeviceGuard g (h->device);
    cudaStream_t st = tpk_stream (h, stream);
    const size_t n = h->n_chan, b = n * 4;
    if (tp_m)  B200M_CUDA (cudaMemcpyAsync (tp_m, h->st.tp_m, b, cudaMemcpyDeviceToHost, st));
    if (tp_p)  B200M_CUDA (cudaMemcpyAsync (tp_p, h->st.tp_p, b, cudaMemcpyDeviceToHost, st));
    if (tp_z1) B200M_CUDA (cudaMemcpyAsync (tp_z1, h->st.tp_z1, b, cudaMemcpyDeviceToHost, st));
    if (tp_z2) B200M_CUDA (cudaMemcpyAsync (tp_z2, h->st.tp_z2, b, cudaMemcpyDeviceToHost, st));
    if (tp_res) B200M_CUDA (cudaMemcpyAsync (tp_res, h->st.tp_res, b, cudaMemcpyDeviceToHost, st));
    if (km8) {
        float* tmp = (float*)malloc (8 * b);
        if (!tmp) return set_err (B200M_E_NOMEM, "host allocation failed");
        const void* src[8] = {h->st.km_z1, h->st.km_z2, h->st.km_rms, h->st.km_peak, h->st.km_fall, h->st.km_cnt, h->st.km_fpp, h->st.km_flag};
        cudaError_t e = cudaSuccess;
        for (int q = 0; q < 8 && e == cudaSuccess; ++q) e = cudaMemcpyAsync (tmp + q * n, src[q], b, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize (st);
        if (e != cudaSuccess) { free (tmp); return cuda_fail (e, "tpk_state", __FILE__, __LINE__); }
        for (size_t i = 0; i < n; ++i)
            for (int q = 0; q < 8; ++q)
                km8[8 * i + q] = (q >= 5) ? (float)((const int*)(tmp + q * n))[i] : tmp[q * n + i];
        free (tmp);
    }
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

// timeline of the slab pipeline's launches (B200M_TPK_TIMELINE=1): n slots of {first CTA start, last CTA end} in globaltimer ns
int b200m_tpk_debug_timeline (b200m_tpk* h, unsigned long long* out, int n)
{
    if (!h || !h->d_tl) return -1;
    cudaDeviceSynchronize ();
    const int m = n < h->tl_next ? n : h->tl_next;
    memcpy (out, h->d_tl, (size_t)m * 2 * sizeof (unsigned long long));
    return m;
}

int b200m_tpk_debug_capture (b200m_tpk* h, int enable)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    DeviceGuard g (h->device);
    B200M_CUDA (cudaDeviceSynchronize ());
    if (enable && !h->d_dbg) B200M_CUDA (cudaMalloc ((void**)&h->d_dbg, (size_t)h->n_chan * 4 * B200M_MAX_BLOCK * sizeof (float)));
    if (!enable && h->d_dbg) { cudaFree (h->d_dbg); h->d_dbg = nullptr; }
    return 0;
}

int b200m_tpk_debug_upsampled (b200m_tpk* h, uint32_t chan, float* out, uint32_t n_out, void* stream)
{
    if (!h || !out || chan >= h->n_chan || n_out > 4 * B200M_MAX_BLOCK) return set_err (B200M_E_INVAL, "bad argument");
    if (!h->d_dbg) return set_err (B200M_E_INVAL, "debug capture not enabled");
    DeviceGuard g (h->device);
    cudaStream_t st = tpk_stream (h, stream);
    B200M_CUDA (cudaMemcpyAsync (out, h->d_dbg + (size_t)chan * 4 * B200M_MAX_BLOCK, (size_t)n_out * 4, cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

}  // extern "C"
