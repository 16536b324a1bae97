// ebu_kw.cuh — the K-weighting recurrence of the EBU R128 bank (K1's per-channel body), shared by the K1 kernels of ebu.cu
// and the fused K-weighting + true-peak kernel of the EBUr128 cycle (tpk.cu); the cycle's dBTP hold (tpk.cu, r128.cu).
#pragma once
#include <cuda.h>
#include "common.cuh"

namespace b200m {

#ifndef B200M_EBU_TILE
#define B200M_EBU_TILE 64
#endif
#ifndef B200M_EBU_TMA_UNROLL
#define B200M_EBU_TMA_UNROLL 8
#endif
#ifndef B200M_EBU_STAGES
#define B200M_EBU_STAGES 3
#endif
constexpr int EBU_TILE   = B200M_EBU_TILE;   // samples per smem tile (64 or 128)
constexpr int EBU_ROWP   = EBU_TILE + 4;  // padded row pitch (floats): = 4 mod 32 -> LDS.128 conflict free
constexpr int EBU_STAGES = B200M_EBU_STAGES; // cp.async pipeline depth (2 tiles = 128 samples in flight per channel)
static_assert (EBU_TILE == 64 || EBU_TILE == 128, "tile geometry");
constexpr int EBU_WARPS  = 4;             // warps per CTA: one per SM sub-partition, each an independent 32-channel pipeline
constexpr int EBU_WARP_FLOATS = EBU_STAGES * 32 * EBU_ROWP;
constexpr int EBU_SMEM_BYTES = EBU_WARPS * EBU_WARP_FLOATS * 4;
constexpr int EBU_MAXCHUNK = 32;          // chunks (block/fragment edges) handled per K1 launch
constexpr int HIST_PITCH = 752;           // 751 bins padded to a 16-byte multiple

struct EbuCoef { float a0, a1, a2, b1, b2, c3, c4; };

// A weighted bank's channel count and per-channel weights (b200m_ebu_create_weighted): kw_warp's run-time form (NCHAN = 0) reads
// them in chunk_end, once per detect_process() call.  Kernels take it as a __grid_constant__ parameter: g[c] is then an indexed
// parameter-space load, not a local copy.
constexpr int EBU_MAXCH_W = 32;           // a K-weighting warp always holds at least one whole instance
struct EbuGains { int nch; float g[EBU_MAXCH_W]; };

// How K1 cuts a block into detect_process() calls.  fph == nullptr: the warp-uniform chunk list v[0..n) (bit31: the chunk ends a
// 50 ms fragment), for a bank whose instances share one fragment phase.  fph != nullptr: every instance has its own phase
// (fph[i]: the bank time mod fragm at which its clock last started; tmod: the bank time mod fragm at the launch's first frame)
// and the launch covers the whole block.
struct EbuChunks {
    int n;
    uint32_t v[EBU_MAXCHUNK];
    int tmod, fragm;
    const int* fph;
};

// Everything one K1 launch over a whole bank needs: the block's first `nfram` frames, its chunk list and the bank's state arrays.
struct EbuK1Args {
    const float* in; size_t stride; int nchans, nfram;
    EbuCoef cf; EbuChunks ck; float fragm_f;
    float *zst, *frpwr, *fragpw; int n_inst;
};

// The EBUr128 cycle's dBTP hold (src/ebulv2.cc:227-230,360-367) as the true-peak kernels' epilogue sees it: nch channels per
// instance, instance i on channels nch i .. nch i + nch - 1.  tpmax == nullptr: no EBUr128 epilogue.  lin == nullptr (nch = 1, 2, 4:
// an instance never leaves an 8-channel true-peak group): the group folds its instances into tpmax[] itself.  Otherwise (nch = 3, 5
// and every weighted bank: instances straddle groups and host slices) every channel's read() goes to lin[channel] and
// r128_hold_kernel folds them.
struct R128Hold { float* tpmax; float* lin; int nch; };

// coef_to_db (src/ebulv2.cc:227-230) of the larger read() t, then tp_max = max (tp_max, tp)
B200M_DEV void r128_hold (float* tpmax, float t)
{
    const float tp = (t == 0) ? -INFINITY : __double2float_rn (__dmul_rn (20.0, (double)log10f_glibc (t)));
    if (tp > *tpmax) *tpmax = tp;
}

// ---- K1: K-weighting recurrence + per-chunk power sums ------------------------------------
// One warp = 32 consecutive mono channels (lane = channel).  Tiles of [32 ch x 64 samples] are
// copied global->shared with cp.async (each row of the planar input is contiguous, so every
// 16-byte copy is fully coalesced), two tiles in flight behind the one being consumed; lane l
// walks row l with LDS.128, the next float4 always loaded one group ahead (the recurrence is a
// pure dependent chain: an exposed LDS latency costs as much as two samples).
// The kernel is bound by per-warp instruction issue, not HBM (DESIGN.md §3): a CTA therefore
// carries exactly one warp per SM sub-partition.
B200M_DEV void kw_step (float p, const EbuCoef& c, float& z1, float& z2, float& z3, float& z4, float& sj)
{
    // x = p - b1*z1 - b2*z2 + 1e-15f;  y = a0*x + a1*z1 + a2*z2 - c3*z3 - c4*z4   (:321-322)
    float x = __fsub_rn (p, __fmul_rn (c.b1, z1));
    x = __fsub_rn (x, __fmul_rn (c.b2, z2));
    x = __fadd_rn (x, 1e-15f);
    float y = __fadd_rn (__fmul_rn (c.a0, x), __fmul_rn (c.a1, z1));
    y = __fadd_rn (y, __fmul_rn (c.a2, z2));
    y = __fsub_rn (y, __fmul_rn (c.c3, z3));
    y = __fsub_rn (y, __fmul_rn (c.c4, z4));
    z2 = z1; z1 = x;
    z4 = __fadd_rn (z4, z3);
    z3 = __fadd_rn (z3, y);
    sj = __fadd_rn (sj, __fmul_rn (y, y));
}

B200M_DEV uint32_t smem_u32 (const void* p) { return (uint32_t)__cvta_generic_to_shared (p); }

// The recurrence over one block for the 32 channels of a warp; `sg` supplies the tiles (a staging policy: PaddedStage and
// TmaStage in ebu.cu, FusedStage in tpk.cu).  PHASES = false compiles the chunk-list policy alone (ck.fph is ignored).
// NCHAN = 0: a weighted bank, gw->nch channels per instance with the weights gw->g (the instance's lanes are lane - lane % nch ..
// + nch - 1); gw is read only in that form.
// RAG (a ragged block, per-instance phases only): instance i processes only its first rlen[i] frames.  Its end is one more
// candidate of the warp's next cut; there its detect_process() call ends (scrub, channel sum, _frpwr +=, and the fragment if an
// edge falls on it) and its state goes to memory at once.  Past that cut the lane keeps stepping through whatever the input holds
// (no per-sample predicate) but never cuts, emits or stores again; rlen[i] = 0: it never does.
template <int NCHAN, bool PHASES, class Stage, bool RAG = false>
B200M_DEV void kw_warp (Stage& sg, int lane, int k, bool live, int nchans, int nfram, const EbuCoef& cf, const EbuChunks& ck, float fragm_f,
                        float* __restrict__ zst, float* __restrict__ frpwr, float* __restrict__ fragpw, int n_inst, const EbuGains* gw = nullptr,
                        const uint32_t* __restrict__ rlen = nullptr)
{
    static_assert (!RAG || PHASES, "a ragged block runs the per-instance phase policy");
    const int ntiles = (nfram + EBU_TILE - 1) / EBU_TILE;
    float z1 = zst[0 * (size_t)nchans + k], z2 = zst[1 * (size_t)nchans + k];
    float z3 = zst[2 * (size_t)nchans + k], z4 = zst[3 * (size_t)nchans + k];
    const int nch = NCHAN ? NCHAN : gw->nch;
    const int inst = k / nch;
    float fp = frpwr[inst];
    float sj = 0.0f;
    int ci = 0, nfr = 0;
    int cend = (int)(ck.v[0] & 0x7fffffffu);           // end position (exclusive) of the current chunk (warp-uniform)
    bool cfrag = (ck.v[0] >> 31) != 0;
    // per-instance phases: the warp cuts at the nearest of its lanes' own fragment edges and the block end; a lane's
    // detect_process() call ends only at its own edges and the block end (:207-216), so at another lane's edge it carries on
    int mynext = 0x7fffffff;                           // this lane's next own fragment edge
    int myend = 0x7fffffff;                            // RAG: this lane's own block end until its lane has cut there
    if (PHASES && ck.fph) {
        if (live) { int el = (ck.tmod - ck.fph[inst]) % ck.fragm; if (el < 0) el += ck.fragm; mynext = ck.fragm - el; }
        if constexpr (RAG) {
            if (live) { myend = (int)rlen[inst]; if (myend == 0) mynext = myend = 0x7fffffff; }
            cend = min (__reduce_min_sync (0xffffffffu, min (mynext, myend)), nfram);
        }
        else cend = min (__reduce_min_sync (0xffffffffu, mynext), nfram);
    }

    // end of one detect_process() call (:324-335): state scrub, channel sum, _frpwr +=, fragment hand-over (:217-221)
    auto chunk_end = [&] () {
        bool cut = true;
        if constexpr (RAG) { cfrag = mynext == cend; cut = cfrag || cend == myend; }
        else if (PHASES && ck.fph) { cfrag = mynext == cend; cut = cfrag || cend == nfram; }
        float si;
        if constexpr (NCHAN == 0) {
            // si = g0 sj0, then si += g_c sj_c in channel order (:328-330 with the caller's weights; 0 + g0 sj0 is g0 sj0 exactly).
            // nch is warp-uniform: every lane runs every shuffle
            const int lead = lane - lane % nch;
            si = __fmul_rn (gw->g[0], __shfl_sync (0xffffffffu, sj, lead));
            for (int c = 1; c < nch; ++c) si = __fadd_rn (si, __fmul_rn (gw->g[c], __shfl_sync (0xffffffffu, sj, (lead + c) & 31)));
        }
        else if (NCHAN == 1) si = __fmul_rn (2.0f, sj);
        else if (NCHAN == 2) si = __fadd_rn (sj, __shfl_xor_sync (0xffffffffu, sj, 1));   // 1.0f*sjL + 1.0f*sjR
        else {
            // si = sum_i _chan_gain[i] * sj_i in channel order, gains 1 1 1 1.41 1.41 (:29,328-329); the instance's lanes are contiguous
            const int lead = lane - lane % nch;
            si = __fmul_rn (1.0f, __shfl_sync (0xffffffffu, sj, lead));
#pragma unroll
            for (int c = 1; c < NCHAN; ++c) si = __fadd_rn (si, __fmul_rn (c >= 3 ? 1.41f : 1.0f, __shfl_sync (0xffffffffu, sj, (lead + c) & 31)));
        }
        if (cut) {                                     // the channel sums above are shuffles: every lane took part
            z1 = scrub (z1); z2 = scrub (z2); z3 = scrub (z3); z4 = scrub (z4);
            fp = __fadd_rn (fp, si);
            if (cfrag) {
                if (live && (k % nch) == 0) fragpw[(size_t)nfr * n_inst + inst] = __fdiv_rn (fp, fragm_f);
                fp = 1e-30f;
                ++nfr;
                mynext += ck.fragm;
            }
            sj = 0.0f;
            if constexpr (RAG) {
                if (cend == myend) {                   // the instance's process() call ends here: its state is final
                    zst[0 * (size_t)nchans + k] = z1; zst[1 * (size_t)nchans + k] = z2;
                    zst[2 * (size_t)nchans + k] = z3; zst[3 * (size_t)nchans + k] = z4;
                    if ((k % nch) == 0) frpwr[inst] = fp;
                    mynext = myend = 0x7fffffff;
                }
            }
        }
        if constexpr (RAG) cend = cend == nfram ? 0x7fffffff : min (__reduce_min_sync (0xffffffffu, min (mynext, myend)), nfram);
        else if (PHASES && ck.fph) cend = cend == nfram ? 0x7fffffff : min (__reduce_min_sync (0xffffffffu, mynext), nfram);
        else {
            ++ci;
            if (ci < ck.n) { cend = (int)(ck.v[ci] & 0x7fffffffu); cfrag = (ck.v[ci] >> 31) != 0; }
            else cend = 0x7fffffff;
        }
    };

    sg.prologue ();
    for (int t = 0; t < ntiles; ++t) {
        sg.acquire (t);
        int a = t * EBU_TILE;
        const int b = min (a + EBU_TILE, nfram);
        if (b - a == EBU_TILE && cend >= b) {
            // fast path: a whole tile inside one chunk; float4 groups with a one-group register prefetch
            float4 cur = sg.ld4 (t, 0);
#pragma unroll Stage::UNROLL
            for (int q = 0; q < EBU_TILE / 4; ++q) {
                const float4 nxt = sg.ld4 (t, (q + 1) & (EBU_TILE / 4 - 1));
                kw_step (cur.x, cf, z1, z2, z3, z4, sj);
                kw_step (cur.y, cf, z1, z2, z3, z4, sj);
                kw_step (cur.z, cf, z1, z2, z3, z4, sj);
                kw_step (cur.w, cf, z1, z2, z3, z4, sj);
                cur = nxt;
            }
            a = b;
            if (a == cend) chunk_end ();
        } else {
            while (a < b) {
                const int e = min (b, cend);
                int j = a;
                // scalar head up to a 4-aligned position, vector body, scalar tail
                for (; j < e && (j & 3); ++j) kw_step (sg.ld (t, j - t * EBU_TILE), cf, z1, z2, z3, z4, sj);
                for (; j + 4 <= e; j += 4) {
                    const float4 v = sg.ld4_dyn (t, (j - t * EBU_TILE) >> 2);
                    kw_step (v.x, cf, z1, z2, z3, z4, sj);
                    kw_step (v.y, cf, z1, z2, z3, z4, sj);
                    kw_step (v.z, cf, z1, z2, z3, z4, sj);
                    kw_step (v.w, cf, z1, z2, z3, z4, sj);
                }
                for (; j < e; ++j) kw_step (sg.ld (t, j - t * EBU_TILE), cf, z1, z2, z3, z4, sj);
                a = e;
                if (a == cend) chunk_end ();
            }
        }
        sg.release (t);
    }
    sg.drain ();
    if (!RAG && live) {                                // RAG: every live lane stored its state at its own end
        zst[0 * (size_t)nchans + k] = z1; zst[1 * (size_t)nchans + k] = z2;
        zst[2 * (size_t)nchans + k] = z3; zst[3 * (size_t)nchans + k] = z4;
        if ((k % nch) == 0) frpwr[inst] = fp;
    }
}

}  // namespace b200m

// host side, ebu.cu: a [rows x cols] float32 tensor map of the planar input with boxes of box_rows x box_cols floats, zeros outside
// (128B swizzle or none); false when the driver offers no encoder or rejects the geometry
bool ebu_tma_map (CUtensorMap* tm, const float* base, size_t stride, uint32_t rows, uint32_t cols, uint32_t box_cols, uint32_t box_rows, bool swizzle128);
// host side, ebu.cu: are these the reference's weights for nchan = 1..5 (mono {2}, else 1 1 1 1.41 1.41), compared bitwise?  And the
// validation of b200m_ebu_create_weighted's arguments (nchan 1..32, finite gains >= 0, one > 0): 0 or B200M_E_INVAL
bool ebu_default_gains (uint32_t nchan, const float* gains);
int ebu_check_gains (uint32_t nchan, const float* gains);
// host side, ebu.cu: does the next `nfram` frames' chunk list fit ONE K1 launch (EBU_MAXCHUNK chunks)?
extern "C" bool ebu_single_k1 (const b200m_ebu* h, uint32_t nfram);
// host side, ebu.cu: one Ebu_r128_proc::process call of every instance, launched per instance slice (see the definition)
extern "C" int ebu_process_sliced (b200m_ebu* h, const float* d_in, size_t stride, uint32_t nfram, cudaStream_t st, int nsl, const uint32_t* bounds,
                                   cudaEvent_t* ready, int (*after_k1) (void*), void* after_arg, int (*k1_fused) (void*, const b200m::EbuK1Args&),
                                   const uint32_t* len = nullptr, const uint32_t* d_len = nullptr);
// host side, ebu.cu: per-instance lengths of a ragged block (b200m_ebu_process_ragged_*).  ebu_ragged_check: 1 if some len[i] differs
// from nfram, 0 if none does (or len is NULL: the plain call), B200M_E_INVAL if one exceeds nfram.  ebu_upload_len: enqueue the
// copy of len[0 .. n_inst) on st into the bank's device array, which it returns (nullptr on a CUDA error, reported by set_err)
extern "C" int ebu_ragged_check (const b200m_ebu* h, uint32_t nfram, const uint32_t* len);
extern "C" const uint32_t* ebu_upload_len (b200m_ebu* h, const uint32_t* len, cudaStream_t st);
