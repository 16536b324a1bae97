// ebu.cu — EBU R128 loudness bank: kernels K1 (K-weighting + fragment power) and K2 (loudness,
// histograms, gating) and the b200m_ebu_* C ABI.
//
// Replaces LV2M::Ebu_r128_proc (ebumeter/ebu_r128_proc.{h,cc} of the reference) for N independent
// instances.  Nothing here is translated from the reference's control flow: the per-sample loop
// (detect_process, ebu_r128_proc.cc:302-337) becomes one thread per mono channel fed by a
// cp.async shared-memory tile pipeline; the 20 Hz bookkeeping (process/addfrags, :207-260) and
// the histogram statistics (Ebu_r128_hist, :66-150) become one warp per instance that walks the
// 751 bins with ballot/shuffle.  Arithmetic ORDER is the reference's, operation by operation
// (no FMA contraction, IEEE div/sqrt, glibc-exact log10f), because the results feed integer
// histogram bins that must be bit-exact.
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <cmath>
#include <cuda.h>
#include <algorithm>
#include <map>
#include <vector>
#include "common.cuh"
#include "ebu_kw.cuh"

namespace b200m {

// ---- staging policies: how a warp's [32 channels x 64 samples] tiles reach shared memory and how lane = channel reads them ----

// (A) cp.async into row-padded tiles (pitch 68 floats = 4 mod 32: conflict-free LDS.128).  Works for any alignment.
template <bool ALIGNED>
struct PaddedStage {
    static constexpr int UNROLL = 4;
    const float* in; size_t stride; float* tile; const float* src_base; int lane, k0, k_end, nfram, ntiles; bool full_warp;

    B200M_DEV void init (const float* in_, size_t stride_, float* smem_warp, int lane_, int k0_, int k_end_, int nfram_)
    {
        in = in_; stride = stride_; tile = smem_warp; lane = lane_; k0 = k0_; k_end = k_end_; nfram = nfram_;
        ntiles = (nfram + EBU_TILE - 1) / EBU_TILE;
        full_warp = k0 + 32 <= k_end;
        src_base = in + (size_t)min (k0 + lane / (EBU_TILE / 4), k_end - 1) * stride + (lane & (EBU_TILE / 4 - 1)) * 4;
    }
    B200M_DEV void issue (int t)
    {
        if (t < ntiles) {
            float* dst = tile + (t % EBU_STAGES) * (32 * EBU_ROWP);
            const int s0 = t * EBU_TILE;
            constexpr int LPR = EBU_TILE / 4;                    // lanes per row (16-byte pieces), rows per pass = 32 / LPR
            constexpr int RPP = 32 / LPR;
            if (ALIGNED) {
                const int c4 = (lane & (LPR - 1)) * 4;           // column of this lane's 16-byte piece
                const int left = (nfram - (s0 + c4)) * 4;        // bytes still inside the block
                const int nb = left >= 16 ? 16 : (left > 0 ? left : 0);
                if (full_warp) {
                    // rows RPP * i + lane / LPR: one base pointer per lane, a constant row step (all 32 channels exist)
                    const float* sp = nb ? src_base + s0 : in;
                    const size_t step = nb ? RPP * stride : 0;
                    float* d = dst + (lane / LPR) * EBU_ROWP + c4;
#pragma unroll
                    for (int i = 0; i < 32 / RPP; ++i) cp_async16 (d + i * RPP * EBU_ROWP, sp + i * step, nb);
                } else {
#pragma unroll 4
                    for (int i = 0; i < 32 / RPP; ++i) {
                        const int r = RPP * i + lane / LPR;
                        const int kr = min (k0 + r, k_end - 1);
                        const float* src = in + (size_t)kr * stride + s0 + c4;
                        cp_async16 (dst + r * EBU_ROWP + c4, nb ? src : in, nb);
                    }
                }
            } else {
#pragma unroll 4
                for (int r = 0; r < 32; ++r) {
                    const int kr = min (k0 + r, k_end - 1);
#pragma unroll
                    for (int h = 0; h < EBU_TILE / 32; ++h) {
                        const int c = lane + 32 * h;
                        const bool ok = (s0 + c) < nfram;
                        cp_async4 (dst + r * EBU_ROWP + c, ok ? in + (size_t)kr * stride + s0 + c : in, ok ? 4 : 0);
                    }
                }
            }
        }
        cp_async_commit ();
    }
    B200M_DEV void prologue () {
#pragma unroll
        for (int t = 0; t < EBU_STAGES - 1; ++t) issue (t);
    }
    B200M_DEV void acquire (int) { cp_async_wait<EBU_STAGES - 2> (); __syncwarp (); }
    // requested after tile t is consumed, not before (the earlier request competes with the recurrence for issue slots)
    B200M_DEV void release (int t) { __syncwarp (); issue (t + EBU_STAGES - 1); }
    B200M_DEV void drain () { cp_async_wait<0> (); }
    B200M_DEV const float* row (int t) const { return tile + (t % EBU_STAGES) * (32 * EBU_ROWP) + lane * EBU_ROWP; }
    B200M_DEV float4 ld4 (int t, int q) const { return reinterpret_cast<const float4*> (row (t))[q]; }
    B200M_DEV float4 ld4_dyn (int t, int q) const { return ld4 (t, q); }
    B200M_DEV float ld (int t, int e) const { return row (t)[e]; }
};

// (B) TMA: one elected lane asks the copy engine for the warp's tile as two [32 rows x 32 floats] boxes (128-byte rows, 128B
// swizzle) completing on an mbarrier -- no per-lane address arithmetic, no zero-fill logic (out-of-range rows / columns
// read as 0).  The 128B swizzle stores 16-byte chunk c of row r at chunk c ^ (r & 7), so the eight lanes of an LDS.128
// phase (rows r..r+7, same logical chunk) hit eight different bank groups: conflict-free without padding.

struct TmaStage {
    static constexpr int UNROLL = B200M_EBU_TMA_UNROLL;       // 8 float4 = one 128-byte row segment: the swizzled offsets are then compile-time
    static constexpr int STAGE_BYTES = 32 * EBU_TILE * 4;        // 8 KB: two 4 KB boxes
    const CUtensorMap* tmap; uint8_t* tile; uint32_t bar; int lane, k0, ntiles; uint32_t off[4];

    B200M_DEV void init (const CUtensorMap* tm, uint8_t* smem_warp, uint64_t* bars, int lane_, int k0_, int nfram)
    {
        tmap = tm; tile = smem_warp; bar = smem_u32 (bars); lane = lane_; k0 = k0_;
        ntiles = (nfram + EBU_TILE - 1) / EBU_TILE;
#pragma unroll
        for (int j = 0; j < 4; ++j) off[j] = (uint32_t)(lane * 128 + ((j ^ (lane & 7)) << 4));
        if (lane == 0) {
#pragma unroll
            for (int s = 0; s < EBU_STAGES; ++s) asm volatile ("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar + 8 * s), "r"(1));
            asm volatile ("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp ();
    }
    B200M_DEV void issue (int t)
    {
        if (t < ntiles && lane == 0) {
            const int s = t % EBU_STAGES;
            const uint32_t dst = smem_u32 (tile + s * STAGE_BYTES), b = bar + 8 * s;
            asm volatile ("fence.proxy.async.shared::cta;" ::: "memory");        // the slot's previous readers (generic proxy) are done
            asm volatile ("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(b), "r"(STAGE_BYTES) : "memory");
#pragma unroll
            for (int h = 0; h < EBU_TILE / 32; ++h)
                asm volatile ("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                              :: "r"(dst + 4096 * h), "l"(tmap), "r"(t * EBU_TILE + 32 * h), "r"(k0), "r"(b) : "memory");
        }
    }
    B200M_DEV void prologue () {
#pragma unroll
        for (int t = 0; t < EBU_STAGES - 1; ++t) issue (t);
    }
    B200M_DEV void acquire (int t)
    {
        const uint32_t b = bar + 8 * (t % EBU_STAGES), parity = (uint32_t)(t / EBU_STAGES) & 1u;
        uint32_t ok = 0;
        while (!ok) asm volatile ("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(b), "r"(parity) : "memory");
    }
    B200M_DEV void release (int t) { __syncwarp (); issue (t + EBU_STAGES - 1); }
    B200M_DEV void drain () {}
    // float4 group q (0..15) of this lane's row: box q >> 3, logical chunk q & 7 = (q & 3) | (q & 4); (j | 4) ^ m = (j ^ m) ^ 4
    B200M_DEV float4 ld4 (int t, int q) const
    {
        const uint8_t* p = tile + (t % EBU_STAGES) * STAGE_BYTES + (q >> 3) * 4096 + (off[q & 3] ^ ((uint32_t)(q & 4) << 4));
        return *reinterpret_cast<const float4*> (p);
    }
    // run-time q (slow path): the offset is computed, not looked up (off[] stays in registers)
    B200M_DEV float4 ld4_dyn (int t, int q) const
    {
        const uint8_t* p = tile + (t % EBU_STAGES) * STAGE_BYTES + (q >> 3) * 4096 + lane * 128 + (((q & 7) ^ (lane & 7)) << 4);
        return *reinterpret_cast<const float4*> (p);
    }
    B200M_DEV float ld (int t, int e) const
    {
        const uint8_t* p = tile + (t % EBU_STAGES) * STAGE_BYTES + (e >> 5) * 4096 + lane * 128 + ((((e >> 2) & 7) ^ (lane & 7)) << 4) + (e & 3) * 4;
        return *reinterpret_cast<const float*> (p);
    }
};

// PHASES: the bank's instances have several fragment phases (ck.fph); without it the chunk-list policy is compiled alone.
// RAG (with PHASES): a ragged block, instance i's rows are read for their first rlen[i] frames only (kw_warp); rlen is not read otherwise
template <int NCHAN, bool ALIGNED, bool PHASES, bool RAG = false>
__global__ void __launch_bounds__ (EBU_WARPS * 32)
ebu_kweight_frag (const float* __restrict__ in, size_t stride, int nchans, int k_first, int k_end, int nfram, EbuCoef cf, EbuChunks ck,
                  float fragm_f, float* __restrict__ zst, float* __restrict__ frpwr, float* __restrict__ fragpw, int n_inst, int pdl_trigger,
                  const uint32_t* __restrict__ rlen)
{
    // channels [k_first, k_end) of the bank's nchans (a slice: *_run_host overlaps the copy of slice s+1 with slice s)
    extern __shared__ __align__ (16) float ebu_smem[];
    // programmatic dependent launch: a kernel launched behind this one with the programmatic-serialization attribute (the
    // true-peak kernel of the EBUr128 cycle, r128.cu) may start as soon as every CTA of this grid is running
    if (pdl_trigger) asm volatile ("griddepcontrol.launch_dependents;");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int CPW = (32 / NCHAN) * NCHAN;          // channels per warp: whole instances only (30 lanes for 3- and 5-channel banks)
    const int k0 = k_first + (blockIdx.x * EBU_WARPS + warp) * CPW;
    if (k0 >= k_end) return;                           // warp-uniform; warps never synchronise with each other
    PaddedStage<ALIGNED> sg;
    sg.init (in, stride, ebu_smem + warp * EBU_WARP_FLOATS, lane, k0, k_end, nfram);
    kw_warp<NCHAN, PHASES, PaddedStage<ALIGNED>, RAG> (sg, lane, min (k0 + lane, k_end - 1) /* tail lanes shadow the last channel (no stores) */,
                                                      lane < CPW && (k0 + lane) < k_end, nchans, nfram, cf, ck, fragm_f, zst, frpwr, fragpw, n_inst, nullptr, rlen);
}

// the same kernel for a weighted bank (b200m_ebu_create_weighted): gw.nch = 1..32 channels per instance, known at run time, a warp
// takes CPW = (32 / nch) nch channels (whole instances), and the channel sum uses the bank's weights gw.g
template <bool ALIGNED, bool PHASES, bool RAG = false>
__global__ void __launch_bounds__ (EBU_WARPS * 32)
ebu_kweight_frag_w (const float* __restrict__ in, size_t stride, int nchans, int k_first, int k_end, int nfram, EbuCoef cf, EbuChunks ck,
                    float fragm_f, float* __restrict__ zst, float* __restrict__ frpwr, float* __restrict__ fragpw, int n_inst, int pdl_trigger,
                    const __grid_constant__ EbuGains gw, const uint32_t* __restrict__ rlen)
{
    extern __shared__ __align__ (16) float ebu_smem[];
    if (pdl_trigger) asm volatile ("griddepcontrol.launch_dependents;");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int cpw = (32 / gw.nch) * gw.nch;
    const int k0 = k_first + (blockIdx.x * EBU_WARPS + warp) * cpw;
    if (k0 >= k_end) return;
    PaddedStage<ALIGNED> sg;
    sg.init (in, stride, ebu_smem + warp * EBU_WARP_FLOATS, lane, k0, k_end, nfram);
    kw_warp<0, PHASES, PaddedStage<ALIGNED>, RAG> (sg, lane, min (k0 + lane, k_end - 1), lane < cpw && (k0 + lane) < k_end,
                                                  nchans, nfram, cf, ck, fragm_f, zst, frpwr, fragpw, n_inst, &gw, rlen);
}

// ---- K1 split over two warps per 32 channels -------------------------------------------------------------------------------
// The recurrence is two biquad-like stages in series (:321-322): stage 1  x = p - b1 z1 - b2 z2 + 1e-15  feeds stage 2
// y = a0 x + a1 z1 + a2 z2 - c3 z3 - c4 z4;  z4 += z3;  z3 += y;  sj += y y.  Each stage is a 16-cycle dependent chain per sample, and
// one warp per SM sub-partition (all a 16384-channel bank offers) cannot hide either behind the other.
// Here warp A runs stage 1 and hands the x stream to warp B (same sub-partition: warps w and w + 4 of the CTA) through a
// double-buffered shared-memory tile; the two chains then interleave on one scheduler.  Every channel sees exactly the same
// operations in the same order as in kw_warp, so the results stay bit-identical.  Named barriers (bar.arrive / bar.sync on 64
// threads) hand the tiles over: a waiting warp is parked by the hardware and takes no issue slots from its partner.
// It knows the warp-uniform chunk list only: a bank whose instances have several fragment phases runs ebu_kweight_frag instead.
// It is slower than the one-warp kernel, so it is opt-in (B200M_EBU_SPLIT=1) and kept for the record: the one-warp kernel is limited
// by the ~21.5 instructions it must ISSUE per sample on its scheduler, not by the 16-cycle chains; a second warp on the SAME scheduler
// adds hand-over instructions and barrier waits without adding issue slots, and every scheduler in use already hosts a warp.
// Only more channels per scheduler help.
constexpr int EBU_SPLIT_PAIRS = 4;
constexpr int EBU_SPLIT_PAIR_FLOATS = (EBU_STAGES + 2) * 32 * EBU_ROWP;
constexpr int EBU_SPLIT_SMEM = EBU_SPLIT_PAIRS * EBU_SPLIT_PAIR_FLOATS * 4;

B200M_DEV void bar_sync64 (int id) { asm volatile ("bar.sync %0, 64;" :: "r"(id) : "memory"); }
B200M_DEV void bar_arrive64 (int id) { asm volatile ("bar.arrive %0, 64;" :: "r"(id) : "memory"); }

B200M_DEV float kw_stage1 (float p, const EbuCoef& c, float& z1, float& z2)
{
    float x = __fsub_rn (p, __fmul_rn (c.b1, z1));
    x = __fsub_rn (x, __fmul_rn (c.b2, z2));
    x = __fadd_rn (x, 1e-15f);
    z2 = z1; z1 = x;
    return x;
}
B200M_DEV void kw_stage2 (float x, const EbuCoef& c, float& z1, float& z2, float& z3, float& z4, float& sj)
{
    float y = __fadd_rn (__fmul_rn (c.a0, x), __fmul_rn (c.a1, z1));       // z1, z2: the two x values before this one
    y = __fadd_rn (y, __fmul_rn (c.a2, z2));
    y = __fsub_rn (y, __fmul_rn (c.c3, z3));
    y = __fsub_rn (y, __fmul_rn (c.c4, z4));
    z2 = z1; z1 = x;
    z4 = __fadd_rn (z4, z3);
    z3 = __fadd_rn (z3, y);
    sj = __fadd_rn (sj, __fmul_rn (y, y));
}

template <int NCHAN, bool ALIGNED>
__global__ void __launch_bounds__ (2 * EBU_SPLIT_PAIRS * 32)
ebu_kweight_split (const float* __restrict__ in, size_t stride, int nchans, int k_first, int k_end, int nfram, EbuCoef cf, EbuChunks ck,
                   float fragm_f, float* __restrict__ zst, float* __restrict__ frpwr, float* __restrict__ fragpw, int n_inst, int pdl_trigger)
{
    extern __shared__ __align__ (16) float ebu_smem[];
    if (pdl_trigger) asm volatile ("griddepcontrol.launch_dependents;");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int pair = warp & (EBU_SPLIT_PAIRS - 1), role = warp / EBU_SPLIT_PAIRS;      // warps w and w + 4 share a sub-partition
    const int k0 = k_first + (blockIdx.x * EBU_SPLIT_PAIRS + pair) * 32;
    if (k0 >= k_end) return;                           // both warps of the pair leave together
    float* pair_smem = ebu_smem + pair * EBU_SPLIT_PAIR_FLOATS;
    float* xt = pair_smem + EBU_STAGES * 32 * EBU_ROWP;   // two x tiles [32][EBU_ROWP]
    const int id_full = pair * 4, id_empty = pair * 4 + 2;
    const int k = min (k0 + lane, k_end - 1);
    const bool live = (k0 + lane) < k_end;
    const int ntiles = (nfram + EBU_TILE - 1) / EBU_TILE;
    float z1 = zst[0 * (size_t)nchans + k], z2 = zst[1 * (size_t)nchans + k];
    int ci = 0;
    int cend = (int)(ck.v[0] & 0x7fffffffu);

    if (role == 0) {
        // ---- warp A: stage 1, input tiles by cp.async, x tiles out
        PaddedStage<ALIGNED> sg;
        sg.init (in, stride, pair_smem, lane, k0, k_end, nfram);
        sg.prologue ();
        for (int t = 0; t < ntiles; ++t) {
            sg.acquire (t);
            if (t >= 2) bar_sync64 (id_empty + (t & 1));              // warp B is done with the x tile written two tiles ago
            float* xrow = xt + (t & 1) * (32 * EBU_ROWP) + lane * EBU_ROWP;
            int a = t * EBU_TILE;
            const int b = min (a + EBU_TILE, nfram);
            if (b - a == EBU_TILE && cend >= b) {
                float4 cur = sg.ld4 (t, 0);
#pragma unroll 4
                for (int q = 0; q < EBU_TILE / 4; ++q) {
                    const float4 nxt = sg.ld4 (t, (q + 1) & (EBU_TILE / 4 - 1));
                    float4 o;
                    o.x = kw_stage1 (cur.x, cf, z1, z2); o.y = kw_stage1 (cur.y, cf, z1, z2);
                    o.z = kw_stage1 (cur.z, cf, z1, z2); o.w = kw_stage1 (cur.w, cf, z1, z2);
                    reinterpret_cast<float4*> (xrow)[q] = o;
                    cur = nxt;
                }
                a = b;
                if (a == cend) { z1 = scrub (z1); z2 = scrub (z2); ++ci; cend = ci < ck.n ? (int)(ck.v[ci] & 0x7fffffffu) : 0x7fffffff; }
            } else {
                while (a < b) {
                    const int e = min (b, cend);
                    for (int j = a; j < e; ++j) xrow[j - t * EBU_TILE] = kw_stage1 (sg.ld (t, j - t * EBU_TILE), cf, z1, z2);
                    a = e;
                    if (a == cend) { z1 = scrub (z1); z2 = scrub (z2); ++ci; cend = ci < ck.n ? (int)(ck.v[ci] & 0x7fffffffu) : 0x7fffffff; }
                }
            }
            bar_arrive64 (id_full + (t & 1));                        // x tile t is complete
            sg.release (t);
        }
        sg.drain ();
        if (live) { zst[0 * (size_t)nchans + k] = z1; zst[1 * (size_t)nchans + k] = z2; }
    } else {
        // ---- warp B: stage 2, power sums, fragment hand-over (the chunk_end of kw_warp)
        float z3 = zst[2 * (size_t)nchans + k], z4 = zst[3 * (size_t)nchans + k];
        const int inst = k / NCHAN;
        float fp = frpwr[inst];
        float sj = 0.0f;
        int nfr = 0;
        bool cfrag = (ck.v[0] >> 31) != 0;
        auto chunk_end = [&] () {
            z1 = scrub (z1); z2 = scrub (z2); z3 = scrub (z3); z4 = scrub (z4);
            float si;
            if (NCHAN == 1) si = __fmul_rn (2.0f, sj);
            else si = __fadd_rn (sj, __shfl_xor_sync (0xffffffffu, sj, 1));
            fp = __fadd_rn (fp, si);
            if (cfrag) {
                if (live && (k % NCHAN) == 0) fragpw[(size_t)nfr * n_inst + inst] = __fdiv_rn (fp, fragm_f);
                fp = 1e-30f;
                ++nfr;
            }
            sj = 0.0f;
            ++ci;
            if (ci < ck.n) { cend = (int)(ck.v[ci] & 0x7fffffffu); cfrag = (ck.v[ci] >> 31) != 0; }
            else cend = 0x7fffffff;
        };
        for (int t = 0; t < ntiles; ++t) {
            bar_sync64 (id_full + (t & 1));
            const float* xrow = xt + (t & 1) * (32 * EBU_ROWP) + lane * EBU_ROWP;
            int a = t * EBU_TILE;
            const int b = min (a + EBU_TILE, nfram);
            if (b - a == EBU_TILE && cend >= b) {
                float4 cur = reinterpret_cast<const float4*> (xrow)[0];
#pragma unroll 4
                for (int q = 0; q < EBU_TILE / 4; ++q) {
                    const float4 nxt = reinterpret_cast<const float4*> (xrow)[(q + 1) & (EBU_TILE / 4 - 1)];
                    kw_stage2 (cur.x, cf, z1, z2, z3, z4, sj); kw_stage2 (cur.y, cf, z1, z2, z3, z4, sj);
                    kw_stage2 (cur.z, cf, z1, z2, z3, z4, sj); kw_stage2 (cur.w, cf, z1, z2, z3, z4, sj);
                    cur = nxt;
                }
                a = b;
                if (a == cend) chunk_end ();
            } else {
                while (a < b) {
                    const int e = min (b, cend);
                    for (int j = a; j < e; ++j) kw_stage2 (xrow[j - t * EBU_TILE], cf, z1, z2, z3, z4, sj);
                    a = e;
                    if (a == cend) chunk_end ();
                }
            }
            if (t + 2 < ntiles) bar_arrive64 (id_empty + (t & 1));       // x tile t may be overwritten (by tile t + 2)
        }
        if (live) {
            zst[2 * (size_t)nchans + k] = z3; zst[3 * (size_t)nchans + k] = z4;
            if ((k % NCHAN) == 0) frpwr[inst] = fp;
        }
    }
}

// the same kernel fed by TMA (16-byte aligned input with a 16-byte multiple row pitch: every bank-sized call in practice); the chunk
// list only, like ebu_kweight_split: a bank with several fragment phases runs ebu_kweight_frag
constexpr int EBU_TMA_SMEM = EBU_WARPS * EBU_STAGES * TmaStage::STAGE_BYTES + EBU_WARPS * EBU_STAGES * 8 + 1024;
template <int NCHAN>
__global__ void __launch_bounds__ (EBU_WARPS * 32)
ebu_kweight_tma (const __grid_constant__ CUtensorMap tmap, int nchans, int k_first, int k_end, int nfram, EbuCoef cf, EbuChunks ck,
                 float fragm_f, float* __restrict__ zst, float* __restrict__ frpwr, float* __restrict__ fragpw, int n_inst, int pdl_trigger)
{
    extern __shared__ uint8_t ebu_smem_raw[];
    if (pdl_trigger) asm volatile ("griddepcontrol.launch_dependents;");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int k0 = k_first + (blockIdx.x * EBU_WARPS + warp) * 32;
    if (k0 >= k_end) return;
    uint8_t* base = ebu_smem_raw + ((1024u - (smem_u32 (ebu_smem_raw) & 1023u)) & 1023u);     // 128B-swizzled boxes want 1 KB alignment (pointer arithmetic
                                                                                          // on the __shared__ symbol keeps the accesses LDS, not generic LD)
    uint64_t* bars = (uint64_t*)(base + EBU_WARPS * EBU_STAGES * TmaStage::STAGE_BYTES) + warp * EBU_STAGES;
    TmaStage sg;
    sg.init (&tmap, base + warp * EBU_STAGES * TmaStage::STAGE_BYTES, bars, lane, k0, nfram);
    // rows >= k_end read as zeros (or as the neighbouring slice's channels): those lanes never store
    kw_warp<NCHAN, false> (sg, lane, min (k0 + lane, k_end - 1), (k0 + lane) < k_end, nchans, nfram, cf, ck, fragm_f, zst, frpwr, fragpw, n_inst);
}

// ---- K2: per-fragment loudness, histograms, gated integration ------------------------------
// wrind: the instance's 64-slot ring write index (_wrind); padded to 32 bytes so that K2a moves it with two 16-byte accesses
struct __align__ (16) EbuCtl { int div1, div2, integr, calc, wrind, pad[3]; };

// Ebu_r128_hist::integrate (:82-102).  `c[t]` holds bin t*32+lane.  Only non-zero bins change the
// running float sum, so the warp walks them in bin order (ballot) and applies the "/= 10 after
// every bin = 99 mod 100" steps in between: identical rounding sequence, ~#non-zero-bins steps.
B200M_DEV float hist_integrate (const int (&c)[24], int i0, const float* bp, int lane)
{
    float s = 0.0f; int n = 0;
    int next_div = i0 - (i0 % 100) + 99;
#pragma unroll
    for (int t = 0; t < 24; ++t) {
        const int bin_l = t * 32 + lane;
        unsigned m = __ballot_sync (0xffffffffu, c[t] != 0 && bin_l >= i0 && bin_l <= 750);
        while (m) {
            const int l = __ffs (m) - 1; m &= m - 1;
            const int kk = __shfl_sync (0xffffffffu, c[t], l);
            const int bin = t * 32 + l;
            while (next_div < bin) { s = __fdiv_rn (s, 10.0f); next_div += 100; }
            s = __fadd_rn (s, __fmul_rn ((float)kk, bp[bin % 100]));
            n += kk;
        }
    }
    while (next_div <= 750) { s = __fdiv_rn (s, 10.0f); next_div += 100; }
    return __fdiv_rn (s, (float)n);
}

B200M_DEV void hist_load (const int* row, int (&c)[24], int lane)
{
#pragma unroll
    for (int t = 0; t < 24; ++t) { const int b = t * 32 + lane; c[t] = (b <= 750) ? row[b] : 0; }
}

// Ebu_r128_hist::calc_integ (:105-125)
B200M_DEV void hist_calc_integ (const int* row, int count, const float* bp, int lane, float& vi, float& th)
{
    if (count < 50) { vi = -200.0f; return; }
    int c[24]; hist_load (row, c, lane);
    float s = hist_integrate (c, 0, bp, lane);
    const float lg = log10f_glibc (s);
    th = __fsub_rn (__fmul_rn (10.0f, lg), 10.0f);
    int k = (int)floorf (__fadd_rn (__fmul_rn (100.0f, lg), 0.5f)) + 600;
    if (k < 0) k = 0;
    s = hist_integrate (c, k, bp, lane);
    vi = __fmul_rn (10.0f, log10f_glibc (s));
}

// Ebu_r128_hist::calc_range (:128-150)
B200M_DEV void hist_calc_range (const int* row, int count, const float* bp, int lane, float& v0, float& v1, float& th)
{
    if (count < 20) { v0 = -200.0f; v1 = -200.0f; return; }
    int c[24]; hist_load (row, c, lane);
    float s = hist_integrate (c, 0, bp, lane);
    const float lg = log10f_glibc (s);
    th = __fsub_rn (__fmul_rn (10.0f, lg), 20.0f);
    // floorf (100 * log10f (s) + 0.5): the 0.5 literal is a double in the reference (:141)
    int k = (int)floorf ((float)((double)__fmul_rn (100.0f, lg) + 0.5)) + 500;
    if (k < 0) k = 0;
    int n = 0;
#pragma unroll
    for (int t = 0; t < 24; ++t) { const int b = t * 32 + lane; if (b >= k && b <= 750) n += c[t]; }
#pragma unroll
    for (int o = 16; o; o >>= 1) n += __shfl_xor_sync (0xffffffffu, n, o);
    const float a = __fmul_rn (0.10f, (float)n), b95 = __fmul_rn (0.95f, (float)n);
    // for (i = k, s = 0; s < a; i++) s += histc[i];
    int i = k; s = 0.0f; bool done = !(s < a);
#pragma unroll
    for (int t = 0; t < 24; ++t) {
        const int bin_l = t * 32 + lane;
        unsigned m = done ? 0u : __ballot_sync (0xffffffffu, c[t] != 0 && bin_l >= k && bin_l <= 750);
        while (m && !done) {
            const int l = __ffs (m) - 1; m &= m - 1;
            s = __fadd_rn (s, (float)__shfl_sync (0xffffffffu, c[t], l));
            if (!(s < a)) { i = t * 32 + l + 1; done = true; }
        }
    }
    // for (j = 750, s = n; s > b; j--) s -= histc[j];
    int j = 750; s = (float)n; done = !(s > b95);
#pragma unroll
    for (int t = 23; t >= 0; --t) {
        const int bin_l = t * 32 + lane;
        unsigned m = done ? 0u : __ballot_sync (0xffffffffu, c[t] != 0 && bin_l <= 750);
        while (m && !done) {
            const int l = 31 - __clz (m); m &= ~(1u << l);
            s = __fsub_rn (s, (float)__shfl_sync (0xffffffffu, c[t], l));
            if (!(s > b95)) { j = t * 32 + l - 1; done = true; }
        }
    }
    v0 = __fdiv_rn ((float)(i - 701), 10.0f);
    v1 = __fdiv_rn ((float)(j - 699), 10.0f);
}

// The loudness log (a PointLog, common.cuh): K2a writes a point's five loudness fields, K2b rewrites three of them after it gates.

// K2a: one THREAD per instance, one completed 50 ms fragment (process :217-243 minus the gated statistics).
// ring layout [64][n_inst] so that lane = instance accesses coalesce; each thread parks its 64-slot ring column
// in shared memory (column private to the thread: no barrier needed) for the two ordered sums.
// Launch `frag` handles row `frag` of fragpw: with one phase for the bank every instance's fragment `frag` of the K1 launch; with
// per-instance phases (fph) each instance's fragment `frag` of the block, if the block of `nfram` frames from bank time tmod has one
// -- in a ragged block (rlen), if the instance's first rlen[i] frames have one.
constexpr int K2A_THREADS = 128;

__global__ void __launch_bounds__ (K2A_THREADS)
ebu_fragment_kernel (int n_inst, int frag, const int* __restrict__ fph, int tmod, int fragm, int nfram, const float* __restrict__ fragpw,
                     float* __restrict__ ring, EbuCtl* __restrict__ ctl, b200m_ebu_result* __restrict__ res, int* __restrict__ histM,
                     int* __restrict__ histS, int* __restrict__ cnt, const uint32_t* __restrict__ rlen, PointLog lg)
{
    __shared__ float sring[64][K2A_THREADS];
    const int tid = threadIdx.x;
    const int i = blockIdx.x * K2A_THREADS + tid;
    if (i >= n_inst) return;
    if (fph) {
        int el = (tmod - fph[i]) % fragm; if (el < 0) el += fragm;
        if (fragm - el + frag * fragm > (rlen ? (int)rlen[i] : nfram)) return;     // the instance's edge `frag` lies beyond its block
    }
    // all 64 ring slots in flight at once (one round of memory latency, not 64): cp.async straight into the column
#pragma unroll
    for (int w = 0; w < 64; ++w) cp_async4 (&sring[w][tid], ring + (size_t)w * n_inst + i, 4);
    cp_async_commit ();
    EbuCtl c = ctl[i];
    b200m_ebu_result r = res[i];
    const float p = fragpw[(size_t)frag * n_inst + i];
    const int wrind = c.wrind;
    cp_async_wait<0> ();
    sring[wrind][tid] = p;                                 // _power[_wrind++] = _frpwr / _fragm (:218)
    ring[(size_t)wrind * n_inst + i] = p;
    const int wr = (wrind + 1) & 63;
    c.wrind = wr;
    r.frag_power = p;
    // addfrags (8), addfrags (60) (:251-260): sequential sums, oldest fragment first
    float s8 = 0.0f, s60 = 0.0f;
    { const int k = (wr - 8) & 63;
#pragma unroll
      for (int q = 0; q < 8; ++q)  s8  = __fadd_rn (s8,  sring[(q + k) & 63][tid]); }
    { const int k = (wr - 60) & 63;
#pragma unroll 10
      for (int q = 0; q < 60; ++q) s60 = __fadd_rn (s60, sring[(q + k) & 63][tid]); }
    float lm = __fadd_rn (-0.6976f, __fmul_rn (10.0f, log10f_glibc (__fdiv_rn (s8, 8.0f))));
    float ls = __fadd_rn (-0.6976f, __fmul_rn (10.0f, log10f_glibc (__fdiv_rn (s60, 60.0f))));
    if (!finitef_ (lm) || lm < -200.0f) lm = -200.0f;      // :224-225
    if (!finitef_ (ls) || ls < -200.0f) ls = -200.0f;
    r.loudness_M = lm; r.loudness_S = ls;
    if (lm > r.maxloudn_M) r.maxloudn_M = lm;
    if (ls > r.maxloudn_S) r.maxloudn_S = ls;
    if (c.integr) {                                         // :228-242
        if (++c.div1 == 2) {                                // Ebu_r128_hist::addpoint (:66-79)
            c.div1 = 0;
            int k = (int)floorf (__fadd_rn (__fmul_rn (10.0f, lm), 700.5f));
            if (k >= 0) {
                if (k > 750) { k = 750; cnt[(size_t)i * 4 + 2]++; }
                histM[(size_t)i * HIST_PITCH + k]++;
                r.hist_M_count = ++cnt[(size_t)i * 4 + 0];
            }
        }
        if (++c.div2 == 10) {
            c.div2 = 0;
            int k = (int)floorf (__fadd_rn (__fmul_rn (10.0f, ls), 700.5f));
            if (k >= 0) {
                if (k > 750) { k = 750; cnt[(size_t)i * 4 + 3]++; }
                histS[(size_t)i * HIST_PITCH + k]++;
                r.hist_S_count = ++cnt[(size_t)i * 4 + 1];
            }
            c.calc = 1;                                     // calc_integ + calc_range follow in K2b
        }
    }
    ctl[i] = c; res[i] = r;
    if (lg.pts) {                                           // the values before this fragment's gating: K2b rewrites I and the range
        const unsigned long long w = lg.written[i];
        const size_t pl = (size_t)lg.cap * n_inst;
        float* p = lg.pts + (size_t)(w % lg.cap) * n_inst + i;
        p[0] = lm; p[pl] = ls; p[2 * pl] = r.integrated; p[3 * pl] = r.range_min; p[4 * pl] = r.range_max;
        lg.written[i] = w + 1;
    }
}

// K2b: one WARP per instance, only launched when the host's phase book-keeping says that some instance
// completed its 10th fragment: calc_integ on hist_M, calc_range on hist_S (:240-241).
constexpr int K2B_WARPS = 4;

__global__ void __launch_bounds__ (K2B_WARPS * 32)
ebu_gate_kernel (int n_inst, EbuCtl* __restrict__ ctl, b200m_ebu_result* __restrict__ res, const int* histM,
                 const int* histS, const int* __restrict__ cnt, const float* __restrict__ bin_power, PointLog lg)
{
    __shared__ float sbp[100];
    for (int q = threadIdx.x; q < 100; q += blockDim.x) sbp[q] = bin_power[q];
    __syncthreads ();
    const int lane = threadIdx.x & 31;
    const int inst = blockIdx.x * K2B_WARPS + (threadIdx.x >> 5);
    if (inst >= n_inst) return;
    if (!ctl[inst].calc) return;
    float vi = res[inst].integrated, th = res[inst].integ_thr;
    float v0 = res[inst].range_min, v1 = res[inst].range_max, rt = res[inst].range_thr;
    hist_calc_integ (histM + (size_t)inst * HIST_PITCH, cnt[(size_t)inst * 4 + 0], sbp, lane, vi, th);
    hist_calc_range (histS + (size_t)inst * HIST_PITCH, cnt[(size_t)inst * 4 + 1], sbp, lane, v0, v1, rt);
    if (lane == 0) {
        res[inst].integrated = vi; res[inst].integ_thr = th;
        res[inst].range_min = v0; res[inst].range_max = v1; res[inst].range_thr = rt;
        ctl[inst].calc = 0;
        // the K2a launch in front of this one set calc and wrote the instance's latest point
        const unsigned long long w = lg.pts ? lg.written[inst] : 0ull;
        if (w) {
            const size_t pl = (size_t)lg.cap * n_inst;
            float* p = lg.pts + (size_t)((w - 1) % lg.cap) * n_inst + inst;
            p[2 * pl] = vi; p[3 * pl] = v0; p[4 * pl] = v1;
        }
    }
}

// a ragged block moves every instance's clock on by its own length, not by the block's nfram: its phase (the bank time at which
// the clock last started) advances by nfram - rlen[i].  Launched behind the block's fragment kernels, which read the old phase.
__global__ void ebu_ragged_clock_kernel (int n_inst, const uint32_t* __restrict__ rlen, int nfram, int fragm, int* __restrict__ fph)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_inst) return;
    fph[i] = (fph[i] + (nfram - (int)rlen[i])) % fragm;
}

// reset / integration control, one thread per instance.  tph >= 0 (cmd 3 only): the instance's clock restarts at bank time tph --
// fragment phase and ring write index -- as in reset(); tph = -1 keeps both (b200m_ebu_clear).  tp_open (the log's dBTP plane is on):
// cmd 3 also drops the true-peak maximum of the instance's open fragment, whose frames the restarted instance no longer meters.
__global__ void ebu_ctl_kernel (int n_inst, int inst_sel, int cmd, int nchan, float* zst, float* frpwr, float* ring,
                                EbuCtl* ctl, b200m_ebu_result* res, int* histM, int* histS, int* cnt, int* fph, int tph, float* tp_open)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_inst || (inst_sel >= 0 && i != inst_sel)) return;
    if (cmd == 0) { ctl[i].integr = 0; return; }            // integr_pause
    if (cmd == 1) { ctl[i].integr = 1; return; }            // integr_start
    // cmd 2: integr_reset (:193-204); cmd 3: reset (:176-190) = integr off + filter/ring clear + integr_reset
    for (int b = 0; b < HIST_PITCH; ++b) { histM[(size_t)i * HIST_PITCH + b] = 0; histS[(size_t)i * HIST_PITCH + b] = 0; }
    for (int b = 0; b < 4; ++b) cnt[(size_t)i * 4 + b] = 0;
    b200m_ebu_result r = res[i];
    r.maxloudn_M = r.maxloudn_S = r.integrated = r.integ_thr = -200.0f;
    r.range_min = r.range_max = r.range_thr = -200.0f;
    r.hist_M_count = r.hist_S_count = 0;
    ctl[i].div1 = ctl[i].div2 = 0; ctl[i].calc = 0;
    if (cmd == 3) {
        ctl[i].integr = 0;
        frpwr[i] = 1e-30f;
        r.loudness_M = r.loudness_S = -200.0f; r.frag_power = 0.0f;
        for (int b = 0; b < 64; ++b) ring[(size_t)b * n_inst + i] = 0.0f;
        const size_t nch = (size_t)n_inst * nchan;
        for (int c = 0; c < nchan; ++c) for (int z = 0; z < 4; ++z) zst[z * nch + (size_t)i * nchan + c] = 0.0f;
        if (tph >= 0) { fph[i] = tph; ctl[i].wrind = 0; }
        if (tp_open) tp_open[i] = 0.0f;
    }
    res[i] = r;
}

// whole-mix histogram sum: grid-stride atomics into one int32[B200M_MIX_WORDS] vector
__global__ void ebu_mix_reduce_kernel (int n_inst, const int* __restrict__ histM, const int* __restrict__ histS,
                                       const int* __restrict__ cnt, int* __restrict__ out)
{
    // blockIdx.x: bin column group (coalescing is across bins); blockIdx.y: slice of the instances.  Integer partial sums are
    // merged with atomicAdd into the zeroed output: order-independent, hence exact.
    const int col = blockIdx.x * blockDim.x + threadIdx.x;    // 0..1507
    if (col >= B200M_MIX_WORDS) return;
    const int per = (n_inst + gridDim.y - 1) / gridDim.y, i0 = blockIdx.y * per, i1 = min (n_inst, i0 + per);
    const int* src; size_t pitch; int c;
    if (col < 752) { src = histM; pitch = HIST_PITCH; c = col; }
    else if (col < 1504) { src = histS; pitch = HIST_PITCH; c = col - 752; }
    else { src = cnt; pitch = 4; c = col - 1504; }
    int acc = 0;
#pragma unroll 8
    for (int i = i0; i < i1; ++i) acc += src[(size_t)i * pitch + c];
    if (acc) atomicAdd (out + col, acc);
}

__global__ void ebu_mix_finish_kernel (const int* __restrict__ mix, const float* __restrict__ bin_power, float* out5)
{
    __shared__ float sbp[100];
    for (int i = threadIdx.x; i < 100; i += blockDim.x) sbp[i] = bin_power[i];
    __syncthreads ();
    const int lane = threadIdx.x;
    float vi = -200.0f, th = -200.0f, v0 = -200.0f, v1 = -200.0f, rt = -200.0f;
    hist_calc_integ (mix, mix[1504], sbp, lane, vi, th);
    hist_calc_range (mix + 752, mix[1505], sbp, lane, v0, v1, rt);
    if (lane == 0) { out5[0] = vi; out5[1] = th; out5[2] = v0; out5[3] = v1; out5[4] = rt; }
}

// Album histogram sums (b200m_ebu_group_reduce).  The host sorts the instances by album into a member list (with each member's album
// beside it) and a CTA takes GRP_CHUNK consecutive members of that list, whatever the album sizes: one album of the whole bank and
// one album per instance both give n / GRP_CHUNK CTAs.  A CTA streams its members' rows (6032 bytes each, one column per thread:
// coalesced) and merges each album's partial sums into the album's zeroed row with integer atomicAdd, skipping zero sums:
// order-independent, hence exact.  Its members are sorted by album, so it flushes once per album it meets.
constexpr int GRP_THREADS = 256, GRP_CHUNK = 16, GRP_BATCH = 4;
constexpr int GRP_COLS = (B200M_MIX_WORDS + GRP_THREADS - 1) / GRP_THREADS;     // columns per thread

__global__ void __launch_bounds__ (GRP_THREADS)
ebu_group_reduce_kernel (const int* __restrict__ histM, const int* __restrict__ histS, const int* __restrict__ cnt,
                         const uint32_t* __restrict__ members, const uint32_t* __restrict__ album, int n_members, int* __restrict__ out)
{
    __shared__ uint32_t mem[GRP_CHUNK], alb[GRP_CHUNK];
    const int first = blockIdx.x * GRP_CHUNK, n = min (GRP_CHUNK, n_members - first);
    if (threadIdx.x < n) { mem[threadIdx.x] = members[first + threadIdx.x]; alb[threadIdx.x] = album[first + threadIdx.x]; }
    __syncthreads ();
    const int* src[GRP_COLS]; int pitch[GRP_COLS]; int acc[GRP_COLS];
#pragma unroll
    for (int j = 0; j < GRP_COLS; ++j) {
        const int col = threadIdx.x + j * GRP_THREADS;
        if (col < 752) { src[j] = histM + col; pitch[j] = HIST_PITCH; }
        else if (col < 1504) { src[j] = histS + (col - 752); pitch[j] = HIST_PITCH; }
        else { src[j] = cnt + (col - 1504); pitch[j] = 4; }
        acc[j] = 0;
    }
    auto flush = [&] (uint32_t a) {
        int* row = out + (size_t)a * B200M_MIX_WORDS;
#pragma unroll
        for (int j = 0; j < GRP_COLS; ++j) {
            const int col = threadIdx.x + j * GRP_THREADS;
            if (col < B200M_MIX_WORDS && acc[j]) atomicAdd (row + col, acc[j]);
            acc[j] = 0;
        }
    };
    // GRP_BATCH members' loads in flight before their sums (a flush between them must not hold back the loads)
    uint32_t cur = alb[0];
    for (int k0 = 0; k0 < n; k0 += GRP_BATCH) {
        int v[GRP_BATCH][GRP_COLS];
#pragma unroll
        for (int q = 0; q < GRP_BATCH; ++q) {
            const size_t m = mem[min (k0 + q, n - 1)];
#pragma unroll
            for (int j = 0; j < GRP_COLS; ++j)
                v[q][j] = (k0 + q < n && threadIdx.x + j * GRP_THREADS < B200M_MIX_WORDS) ? src[j][m * pitch[j]] : 0;
        }
#pragma unroll
        for (int q = 0; q < GRP_BATCH; ++q) {
            if (k0 + q < n && alb[k0 + q] != cur) { flush (cur); cur = alb[k0 + q]; }        // uniform across the CTA
#pragma unroll
            for (int j = 0; j < GRP_COLS; ++j) acc[j] += v[q][j];
        }
    }
    flush (cur);
}

// b200m_ebu_group_finish: one warp per album row, the whole-mix finish of each (rows is not __restrict__: with it ptxas spills)
constexpr int GRP_FIN_WARPS = 4;

__global__ void __launch_bounds__ (GRP_FIN_WARPS * 32)
ebu_group_finish_kernel (int n_groups, const int* rows, const float* __restrict__ bin_power, float* __restrict__ out5)
{
    __shared__ float sbp[100];
    for (int q = threadIdx.x; q < 100; q += blockDim.x) sbp[q] = bin_power[q];
    __syncthreads ();
    const int lane = threadIdx.x & 31;
    const int g = blockIdx.x * GRP_FIN_WARPS + (threadIdx.x >> 5);
    if (g >= n_groups) return;
    const int* row = rows + (size_t)g * B200M_MIX_WORDS;
    float vi = -200.0f, th = -200.0f, v0 = -200.0f, v1 = -200.0f, rt = -200.0f;
    hist_calc_integ (row, row[1504], sbp, lane, vi, th);
    hist_calc_range (row + 752, row[1505], sbp, lane, v0, v1, rt);
    if (lane == 0) { float* o = out5 + (size_t)g * 5; o[0] = vi; o[1] = th; o[2] = v0; o[3] = v1; o[4] = rt; }
}

}  // namespace b200m

using namespace b200m;

// ---------------------------------------------------------------------------- host side
// cuTensorMapEncodeTiled through the runtime's driver entry point (libcuda is not linked)
typedef CUresult (*TmaEncodeFn) (CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                 CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static TmaEncodeFn tma_encoder ()
{
    static TmaEncodeFn fn = [] () -> TmaEncodeFn {
        void* p = nullptr; cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint ("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
        return (TmaEncodeFn)p;
    }();
    return fn;
}
bool ebu_tma_map (CUtensorMap* tm, const float* base, size_t stride, uint32_t rows, uint32_t cols, uint32_t box_cols, uint32_t box_rows, bool swizzle128)
{
    if (!tma_encoder ()) return false;
    const cuuint64_t gdim[2] = {cols, rows}; const cuuint64_t gstr[1] = {(cuuint64_t)stride * sizeof (float)};
    const cuuint32_t box[2] = {box_cols, box_rows}, es[2] = {1, 1};
    return tma_encoder () (tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*> (base), gdim, gstr, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// [rows x cols] float32 view of the planar input for K1: boxes of 32 rows x 32 floats, 128B swizzle, zeros outside
static bool tma_input_map (CUtensorMap* tm, const float* base, size_t stride, uint32_t rows, uint32_t cols)
{
    return ebu_tma_map (tm, base, stride, rows, cols, 32, 32, true);
}

// The bank's sample clock T is kept on the host as tmod = T mod fragm.  Instance i's 50 ms fragment clock last started at bank
// time fph[i] (mod fragm): a device value mirrored on the host in ph[i], written by the control kernel (the clock restarts) and by
// ebu_ragged_clock_kernel (a ragged block: the instance's clock ran rlen[i] frames, not nfram).  Its next edge lies
// fragm - ((T - fph[i]) mod fragm) frames ahead.
struct EbuPhase { int n = 0, G = 0; int cnt10[10] = {0}; };   // one phase class: members, fragment counter mod 10, S-period census

struct b200m_ebu {
    int device; uint32_t n_inst, nchan; float fsamp; int fragm;
    bool weighted = false; EbuGains gw = {};   // b200m_ebu_create_weighted with other than the default weights: ebu_kweight_frag_w
    int tmod = 0;                        // bank time mod fragm
    int fragrows = EBU_MAXCHUNK;         // rows of d_fragpw: the most fragments one K1 launch completes per instance
    EbuCoef cf;
    float *d_z = nullptr, *d_frpwr = nullptr, *d_fragpw = nullptr, *d_ring = nullptr, *d_binpow = nullptr, *d_out5 = nullptr;
    EbuCtl* d_ctl = nullptr; b200m_ebu_result* d_res = nullptr;
    int *d_histM = nullptr, *d_histS = nullptr, *d_cnt = nullptr, *d_fph = nullptr;
    // the loudness log (b200m_ebu_log_enable), off while ring.log.pts is null: the planes and written counters K2a / K2b update
    PointRing ring;
    // the log's dBTP plane (b200m_r128_log_enable), off while tp.fmax is null
    EbuTpPlane tp = {};
    void log_free () {
        ring.release ();
        cudaFree (tp.fmax); cudaFree (tp.fph0); cudaFree (tp.open); cudaFree (tp.filled);
        tp = {};
    }
    BankPath path;
    // the path of the EBUr128 bank this bank belongs to (ebu_follow), nullptr for a bank of its own: that bank drives this one's
    // kernels on its streams, so this bank's getters, controls and log calls resolve their stream through its path
    const BankPath* owner = nullptr;
    cudaStream_t stream (void* caller) const { return (owner ? owner : &path)->stream (caller); }
    bool use_tma = false;                // K1 tiles by TMA (opt-in, 16-byte aligned input only) instead of cp.async
    bool split = false;                  // K1 as two warps per 32 channels (ebu_kweight_split), opt-in with B200M_EBU_SPLIT=1: measured slower, see the kernel
    // Host mirror of every instance's S-histogram period (_div2, :234-241), kept in O(1) per fragment and phase class: the
    // instances that share a fragment phase form a class whose G counts their fragments; an integrating instance has
    // div2 = (G - base) mod 10 and cnt10[r] = number of integrating members with base = r.  The gated-statistics kernel (K2b)
    // is launched only behind fragments where some class has cnt10[G] > 0.  The classes are ordered by phase.
    std::vector<uint8_t> integ, base, frozen; std::vector<int> ph;
    std::map<int, EbuPhase> cls;
    std::vector<int> nf;                 // per class: fragments it completes in the block being launched (scratch)
    // a ragged block (b200m_ebu_process_ragged_*, b200m_r128_run_ragged_*): the upload of its per-instance lengths, and the instances
    // whose length differs from nfram (scratch: index, fragments in the block, S-period position div2)
    RaggedLen rag;
    // album reduce (b200m_ebu_group_reduce): the member list (GroupList, common.cuh); the finish's device output, grown on demand
    GroupList grp;
    float* d_grp5 = nullptr; uint32_t grp5_cap = 0;
    struct Rag { uint32_t i; int nf, d2; };
    std::vector<Rag> rg;
    void phase_reset () {
        integ.assign (n_inst, 0); base.assign (n_inst, 0); frozen.assign (n_inst, 0); ph.assign (n_inst, tmod);
        cls.clear (); cls[tmod].n = (int)n_inst;
    }
    void phase_ctl (int32_t inst, int cmd) {
        for (uint32_t i = 0; i < n_inst; ++i) {
            if (inst >= 0 && (uint32_t)inst != i) continue;
            EbuPhase& c = cls[ph[i]];
            if (cmd == 0 && integ[i]) { frozen[i] = (uint8_t)((c.G - base[i] + 10) % 10); c.cnt10[base[i]]--; integ[i] = 0; }
            else if (cmd == 1 && !integ[i]) { base[i] = (uint8_t)((c.G - frozen[i] + 10) % 10); c.cnt10[base[i]]++; integ[i] = 1; }
            else if (cmd == 2) { if (integ[i]) { c.cnt10[base[i]]--; base[i] = (uint8_t)c.G; c.cnt10[base[i]]++; } else frozen[i] = 0; }
        }
    }
    // reset() of one instance: integration off, div counters cleared, its clock restarted now
    void phase_restart (uint32_t i) {
        phase_ctl ((int32_t)i, 0); phase_ctl ((int32_t)i, 2);
        auto it = cls.find (ph[i]);
        if (--it->second.n == 0) cls.erase (it);
        ph[i] = tmod; cls[tmod].n++;
    }
    // fragments that instances of phase p complete in the next nfram frames
    int frags_in (int p, uint32_t nfram) const {
        int el = (tmod - p) % fragm; if (el < 0) el += fragm;
        const int e0 = fragm - el;
        return e0 <= (int)nfram ? 1 + ((int)nfram - e0) / fragm : 0;
    }
    int frcnt_of (int p) const { int el = (tmod - p) % fragm; if (el < 0) el += fragm; return fragm - el; }
    static bool phase_tick (EbuPhase& c) { c.G = (c.G + 1) % 10; return c.cnt10[c.G] > 0; }   // one fragment of the class: does anyone wrap?
    // A ragged block: instance i with len[i] != nfram completes another number of fragments than its class, so it leaves the class
    // for the block and is ticked on its own, its S-period position kept as div2 = (G - base) mod 10 (integrating) or in frozen
    // (paused).  O(classes + such instances) besides the scan of len.
    void ragged_leave (const uint32_t* len, uint32_t nfram) {
        rg.clear ();
        for (uint32_t i = 0; i < n_inst; ++i) {
            if (len[i] == nfram) continue;
            auto it = cls.find (ph[i]);
            EbuPhase& c = it->second;
            int d2 = 0;
            if (integ[i]) { d2 = (c.G - base[i] + 10) % 10; c.cnt10[base[i]]--; }
            rg.push_back ({i, frags_in (ph[i], len[i]), d2});
            if (--c.n == 0) cls.erase (it);
        }
    }
    // ... one fragment f of the block for the instances that left: does an integrating one wrap its S period?
    bool ragged_tick (int f) {
        bool wrap = false;
        for (auto& r : rg)
            if (f < r.nf && integ[r.i]) { r.d2 = (r.d2 + 1) % 10; wrap |= r.d2 == 0; }
        return wrap;
    }
    // ... and after it each joins the class of its new phase ph + nfram - len (ebu_ragged_clock_kernel), keeping its S-period position
    void ragged_join (const uint32_t* len, uint32_t nfram) {
        for (const auto& r : rg) {
            const uint32_t i = r.i;
            ph[i] = (int)(((uint32_t)ph[i] + (nfram - len[i])) % (uint32_t)fragm);
            EbuPhase& c = cls[ph[i]];
            c.n++;
            if (integ[i]) { base[i] = (uint8_t)((c.G - r.d2 + 10) % 10); c.cnt10[base[i]]++; }
        }
        rg.clear ();
    }
};

// Host-side coefficient design; restates Ebu_r128_proc::detect_init (ebu_r128_proc.cc:263-293).
// Same literals and the same float expression types (tan on a float argument is the float
// overload in C++), evaluated with the host libm, so every coefficient is bitwise the oracle's.
static void ebu_design (float fsamp, EbuCoef& k)
{
    const float rt = 1 / tanf (4712.3890f / fsamp);
    const float wa = rt / 1.12201f, wb = rt * 1.12201f;
    const float u = 1.4085f + 210.0f / fsamp;
    const float pa = u * wa, pb = wa * wa, pc = u * wb, pd = wb * wb;
    const float den = 1 + pa + pb;
    k.a0 = (1 + pc + pd) / den;
    k.a1 = (2 - 2 * pd) / den;
    k.a2 = (1 - pc + pd) / den;
    k.b1 = (2 - 2 * pb) / den;
    k.b2 = (1 - pa + pb) / den;
    const float q = 48.0f / fsamp;
    float ha = 4.9886075f * q, hb = 6.2298014f * q * q;
    const float hden = 1 + ha + hb;
    ha *= 2 / hden; hb *= 4 / hden;
    k.c3 = ha + hb; k.c4 = hb;
    const float g = 1.004995f / hden;
    k.a0 *= g; k.a1 *= g; k.a2 *= g;
}

static int ebu_ctl (b200m_ebu* h, int32_t inst, int cmd, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    if (inst >= (int32_t)h->n_inst) return set_err (B200M_E_INVAL, "instance %d out of range", inst);
    DeviceGuard g (h->device);
    if (cmd == 3) { if (inst < 0) h->phase_reset (); else h->phase_restart ((uint32_t)inst); }
    else h->phase_ctl (inst, cmd);
    // after process_host the bank runs on its own stream: a control on any other stream would race with the kernels in flight
    ebu_ctl_kernel<<<(h->n_inst + 127) / 128, 128, 0, h->stream (stream)>>> (
        (int)h->n_inst, inst, cmd, (int)h->nchan, h->d_z, h->d_frpwr, h->d_ring, h->d_ctl, h->d_res, h->d_histM, h->d_histS, h->d_cnt,
        h->d_fph, cmd == 3 ? h->tmod : -1, h->tp.open);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

extern "C" {

int b200m_design_ebu (float fsamp, float o[7])
{
    if (!o || !(fsamp >= 1000.0f)) return set_err (B200M_E_INVAL, "bad argument");
    EbuCoef k; ebu_design (fsamp, k);
    o[0] = k.a0; o[1] = k.a1; o[2] = k.a2; o[3] = k.b1; o[4] = k.b2; o[5] = k.c3; o[6] = k.c4;
    return 0;
}

}  // extern "C"

bool ebu_default_gains (uint32_t nchan, const float* gains)
{
    static const float dflt[5] = {1.0f, 1.0f, 1.0f, 1.41f, 1.41f};          // ebu_r128_proc.cc:29; mono: 2 * sj (:327)
    if (nchan < 1 || nchan > 5) return false;
    if (nchan == 1) { const float two = 2.0f; return memcmp (gains, &two, 4) == 0; }
    return memcmp (gains, dflt, 4 * nchan) == 0;
}

int ebu_check_gains (uint32_t nchan, const float* gains)
{
    if (nchan < 1 || nchan > (uint32_t)EBU_MAXCH_W) return set_err (B200M_E_INVAL, "nchan %u outside 1..%d", nchan, EBU_MAXCH_W);
    if (!gains) return set_err (B200M_E_INVAL, "NULL gains");
    bool any = false;
    for (uint32_t c = 0; c < nchan; ++c) {
        if (!std::isfinite (gains[c]) || gains[c] < 0.0f) return set_err (B200M_E_INVAL, "gain %u is not finite and >= 0", c);
        any |= gains[c] > 0.0f;
    }
    return any ? 0 : set_err (B200M_E_INVAL, "every gain is zero");
}

// gains == nullptr: the default weights of a 1..5-channel bank (the compile-time K1 instantiations); otherwise a weighted bank
// K1 selectors: the launch in ebu_process_sliced and ebu_create's attributes both go through them.  With several fragment phases
// or a ragged block (PHASES, RAG) every lane cuts at its own instance's fragment edges; a ragged block always has phases.
// ebu_kweight_frag of an unweighted bank (1..5 channels per instance)
static auto ebu_k1_for (int nchan, bool al, bool phases, bool rag)
{
    return with_int<1, 2, 3, 4, 5> (nchan, [&] (auto NC) {
        return with_bools ([&] (auto AL, auto PH, auto RG) { return ebu_kweight_frag<NC, AL, PH || RG, RG>; }, al, phases, rag);
    });
}
// ebu_kweight_frag_w of a weighted bank (the run-time channel count)
static auto ebu_k1w_for (bool al, bool phases, bool rag)
{
    return with_bools ([] (auto AL, auto PH, auto RG) { return ebu_kweight_frag_w<AL, PH || RG, RG>; }, al, phases, rag);
}
// the opt-in variants of 1..2 channels per instance, one phase class: TMA staging and split K-weighting roles
static auto ebu_k1t_for (int nchan) { return with_int<1, 2> (nchan, [] (auto NC) { return ebu_kweight_tma<NC>; }); }
static auto ebu_k1s_for (int nchan, bool al)
{
    return with_int<1, 2> (nchan, [&] (auto NC) { return with_bools ([&] (auto AL) { return ebu_kweight_split<NC, AL>; }, al); });
}

static int ebu_create (b200m_ebu** out, int device, uint32_t n_inst, uint32_t nchan, float fsamp, const float* gains)
{
    if (n_inst == 0 || !(fsamp >= 1000.0f)) return set_err (B200M_E_INVAL, "bad n_inst/fsamp");
    if (b200m_device_count () <= 0) return set_err (B200M_E_NODEVICE, "no CUDA device: b200meters has no CPU path");
    DeviceGuard g (device);
    if (!g.ok) return set_err (B200M_E_NODEVICE, "cannot select CUDA device %d", device);
    b200m_ebu* h = new (std::nothrow) b200m_ebu;
    if (!h) return set_err (B200M_E_NOMEM, "host allocation failed");
    h->device = device; h->n_inst = n_inst; h->nchan = nchan; h->fsamp = fsamp;
    if (gains) { h->weighted = true; h->gw.nch = (int)nchan; memcpy (h->gw.g, gains, 4 * nchan); }
    h->fragm = (int)fsamp / 20;                     // :170
    // with per-instance phases one K1 launch covers a whole block (a split would add a cut the reference does not make)
    h->fragrows = std::max<int> (EBU_MAXCHUNK, (int)(B200M_MAX_BLOCK / (uint32_t)h->fragm) + 2);
    ebu_design (fsamp, h->cf);
    const size_t nch = (size_t)n_inst * nchan;
    float bp[100];
    for (int i = 0; i < 100; ++i) bp[i] = powf (10.0f, i / 100.0f);   // Ebu_r128_hist::initstat (:54-63)
    cudaError_t e = cudaSuccess;
    auto A = [&] (void** p, size_t bytes) { if (e == cudaSuccess) { e = cudaMalloc (p, bytes); if (e == cudaSuccess) e = cudaMemset (*p, 0, bytes); } };
    A ((void**)&h->d_z, 4 * nch * sizeof (float));
    A ((void**)&h->d_frpwr, n_inst * sizeof (float));
    A ((void**)&h->d_fragpw, (size_t)h->fragrows * n_inst * sizeof (float));
    A ((void**)&h->d_ring, (size_t)64 * n_inst * sizeof (float));
    A ((void**)&h->d_binpow, 100 * sizeof (float));
    A ((void**)&h->d_out5, 8 * sizeof (float));
    A ((void**)&h->d_ctl, n_inst * sizeof (EbuCtl));
    A ((void**)&h->d_res, n_inst * sizeof (b200m_ebu_result));
    A ((void**)&h->d_histM, (size_t)HIST_PITCH * n_inst * sizeof (int));
    A ((void**)&h->d_histS, (size_t)HIST_PITCH * n_inst * sizeof (int));
    A ((void**)&h->d_cnt, (size_t)4 * n_inst * sizeof (int));
    A ((void**)&h->d_fph, n_inst * sizeof (int));
    if (e == cudaSuccess) e = cudaMemcpy (h->d_binpow, bp, sizeof (bp), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags (&h->path.own, cudaStreamNonBlocking);
    // K1 carries 102 KB of dynamic shared memory per CTA
    // ... and asks for the largest shared-memory carveout: with the default the driver configures the SM for just what this kernel
    // needs (132 KB), which leaves room for ONE CTA of the true-peak kernel that is meant to share the SM with it (r128.cu)
    auto attrs = [&] (auto k, int smem) {
        if (e == cudaSuccess) e = cudaFuncSetAttribute (k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e == cudaSuccess) e = cudaFuncSetAttribute (k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    };
    for (const bool al : {false, true})
        for (const bool ph : {false, true})
            for (const bool rag : {false, true}) {
                for (int nc = 1; nc <= 5; ++nc) attrs (ebu_k1_for (nc, al, ph, rag), EBU_SMEM_BYTES);
                if (gains) attrs (ebu_k1w_for (al, ph, rag), EBU_SMEM_BYTES);
            }
    // TMA staging is bit-identical and removes ~120 address instructions per tile, but is no faster standalone and slower inside the
    // EBUr128 cycle (the mbarrier try_wait spin takes issue slots from the co-running true-peak kernel, a scoreboard wait does not):
    // opt-in with B200M_EBU_TMA=1
    for (int nc = 1; nc <= 2; ++nc) {
        attrs (ebu_k1t_for (nc), EBU_TMA_SMEM);
        for (const bool al : {false, true}) attrs (ebu_k1s_for (nc, al), EBU_SPLIT_SMEM);
    }
    if (const char* v = getenv ("B200M_EBU_SPLIT")) h->split = atoi (v) != 0;
    h->use_tma = false;
    if (const char* v = getenv ("B200M_EBU_TMA")) h->use_tma = atoi (v) != 0 && tma_encoder () != nullptr;
    if (e != cudaSuccess) { int rc = cuda_fail (e, "ebu_create allocations", __FILE__, __LINE__); b200m_ebu_destroy (h); return rc; }
    h->phase_reset ();
    int rc = b200m_ebu_reset (h, -1, nullptr);       // constructor + init() end in reset() (:153-173)
    if (rc == 0 && cudaDeviceSynchronize () != cudaSuccess) rc = set_err (B200M_E_CUDA, "reset kernel failed");
    if (rc) { b200m_ebu_destroy (h); return rc; }
    *out = h;
    return 0;
}

extern "C" {

int b200m_ebu_create (b200m_ebu** out, int device, uint32_t n_inst, uint32_t nchan, float fsamp)
{
    if (!out) return set_err (B200M_E_INVAL, "NULL out pointer");
    *out = nullptr;
    if (nchan < 1 || nchan > 5) return set_err (B200M_E_INVAL, "nchan %u outside 1..5", nchan);
    return ebu_create (out, device, n_inst, nchan, fsamp, nullptr);
}

int b200m_ebu_create_weighted (b200m_ebu** out, int device, uint32_t n_inst, uint32_t nchan, const float* gains, float fsamp)
{
    if (!out) return set_err (B200M_E_INVAL, "NULL out pointer");
    *out = nullptr;
    if (int rc = ebu_check_gains (nchan, gains)) return rc;
    return ebu_create (out, device, n_inst, nchan, fsamp, ebu_default_gains (nchan, gains) ? nullptr : gains);
}

// ITU-R BS.1770-4 channel weights from loudspeaker positions: 1.41 for |elevation| < 30 degrees and 60 <= |azimuth| <= 120 degrees
// (azimuth taken modulo 360 into -180 .. 180), 1.0 otherwise.  Host only.
int b200m_bs1770_weights (uint32_t n, const float* azimuth_deg, const float* elevation_deg, float* gains)
{
    if (n && (!azimuth_deg || !elevation_deg || !gains)) return set_err (B200M_E_INVAL, "NULL argument");
    for (uint32_t c = 0; c < n; ++c)
        if (!std::isfinite (azimuth_deg[c]) || !std::isfinite (elevation_deg[c])) return set_err (B200M_E_INVAL, "position %u is not finite", c);
    for (uint32_t c = 0; c < n; ++c) {
        double az = fmod ((double)azimuth_deg[c], 360.0);
        if (az > 180.0) az -= 360.0;
        else if (az < -180.0) az += 360.0;
        az = fabs (az);
        gains[c] = (fabs ((double)elevation_deg[c]) < 30.0 && az >= 60.0 && az <= 120.0) ? 1.41f : 1.0f;
    }
    return 0;
}

int b200m_ebu_destroy (b200m_ebu* h)
{
    if (!h) return 0;
    DeviceGuard g (h->device);
    cudaDeviceSynchronize ();
    cudaFree (h->d_z); cudaFree (h->d_frpwr); cudaFree (h->d_fragpw); cudaFree (h->d_ring); cudaFree (h->d_binpow);
    cudaFree (h->d_out5); cudaFree (h->d_ctl); cudaFree (h->d_res); cudaFree (h->d_histM); cudaFree (h->d_histS); cudaFree (h->d_cnt); cudaFree (h->d_fph);
    h->log_free ();
    h->rag.release ();
    h->grp.release (); cudaFree (h->d_grp5);
    h->path.release ();
    delete h;
    return 0;
}

int b200m_ebu_reset (b200m_ebu* h, int32_t inst, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    if (inst < -1) return set_err (B200M_E_INVAL, "instance %d out of range", inst);
    return ebu_ctl (h, inst, 3, stream);         // the instance's (every instance's) clock restarts at the current bank time
}
int b200m_ebu_clear (b200m_ebu* h, int32_t inst, void* stream)
{
    // what reset() does to ONE instance -- integration off, filter states, 64-fragment ring, loudness values, histograms -- without
    // restarting its 50 ms fragment clock
    if (!h || inst < 0 || inst >= (int32_t)h->n_inst) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    h->phase_ctl (inst, 0); h->phase_ctl (inst, 2);
    ebu_ctl_kernel<<<(h->n_inst + 127) / 128, 128, 0, h->stream (stream)>>> (
        (int)h->n_inst, inst, 3, (int)h->nchan, h->d_z, h->d_frpwr, h->d_ring, h->d_ctl, h->d_res, h->d_histM, h->d_histS, h->d_cnt,
        h->d_fph, -1, h->tp.open);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}
int b200m_ebu_integr_start (b200m_ebu* h, int32_t inst, void* stream) { return ebu_ctl (h, inst, 1, stream); }
int b200m_ebu_integr_pause (b200m_ebu* h, int32_t inst, void* stream) { return ebu_ctl (h, inst, 0, stream); }
int b200m_ebu_integr_reset (b200m_ebu* h, int32_t inst, void* stream) { return ebu_ctl (h, inst, 2, stream); }

// Cut the next `rem` frames at fragment edges, at most EBU_MAXCHUNK pieces (one K1 launch, :212-216), advancing the fragment
// counter `frcnt`; returns the frames the chunk list covers.
static uint32_t ebu_plan_chunks (int& frcnt, int fragm, uint32_t rem, EbuChunks& ck, int& nfrag)
{
    ck.n = 0; nfrag = 0;
    uint32_t pos = 0;
    while (pos < rem && ck.n < EBU_MAXCHUNK) {
        const uint32_t left = rem - pos;
        const uint32_t k = (uint32_t)frcnt < left ? (uint32_t)frcnt : left;
        pos += k; frcnt -= (int)k;
        uint32_t v = pos;
        if (frcnt == 0) { v |= 0x80000000u; frcnt = fragm; ++nfrag; }
        ck.v[ck.n++] = v;
    }
    return pos;
}

bool ebu_single_k1 (const b200m_ebu* h, uint32_t nfram)
{
    if (h->cls.size () > 1) return true;             // per-instance phases: always one launch per block
    int frcnt = h->frcnt_of (h->cls.begin ()->first), nfrag; EbuChunks ck;
    return ebu_plan_chunks (frcnt, h->fragm, nfram, ck, nfrag) == nfram;
}

// One Ebu_r128_proc::process call for every instance.  `nsl` instance slices [bounds[s], bounds[s+1]) are launched
// separately, slice s after event ready[s] (the host->device copy of its rows) when `ready` is given; the
// fragment/gating kernels run once, after the last slice.
// `k1_fused`, when given (one slice, a block whose chunk list fits one launch: ebu_single_k1), launches a kernel that does
// K1's work over the whole bank in its place; `after_k1` is enqueued right behind the first K1 launch.
// `len` (host) / `d_len` (its copy on the device, ebu_lens): a ragged block, instance i processes its first len[i] frames (some
// len[i] differs from nfram: ragged_check); nullptr: every instance processes nfram.
int ebu_process_sliced (b200m_ebu* h, const float* d_in, size_t stride, uint32_t nfram, cudaStream_t st,
                        int nsl, const uint32_t* bounds, cudaEvent_t* ready, int (*after_k1) (void*), void* after_arg,
                        int (*k1_fused) (void*, const EbuK1Args&), const uint32_t* len, const uint32_t* d_len)
{
    const int nch = (int)(h->n_inst * h->nchan);
    const bool aligned = ((uintptr_t)d_in % 16 == 0) && (stride % 4 == 0);
    // one phase class: the warp-uniform chunk list, split over launches of at most EBU_MAXCHUNK chunks; several, or a ragged block:
    // one launch per block, every lane cutting at its own instance's fragment edges (and its own end)
    if (d_len) h->ragged_leave (len, nfram);
    const bool multi = d_len || h->cls.size () > 1;
    int frcnt = multi ? 0 : h->frcnt_of (h->cls.begin ()->first);
    uint32_t done = 0;
    while (done < nfram) {
        EbuChunks ck; int nfrag = 0;
        uint32_t pos = nfram;
        ck.tmod = h->tmod; ck.fragm = h->fragm; ck.fph = nullptr;
        if (multi) {
            ck.n = 0; ck.v[0] = 0; ck.fph = h->d_fph;
            h->nf.clear ();
            for (const auto& c : h->cls) { h->nf.push_back (h->frags_in (c.first, nfram)); nfrag = std::max (nfrag, h->nf.back ()); }
            for (const auto& r : h->rg) nfrag = std::max (nfrag, r.nf);
        }
        else pos = ebu_plan_chunks (frcnt, h->fragm, nfram - done, ck, nfrag);
        const float* src = d_in + done;
        const bool fused = k1_fused && !d_len && done == 0 && pos == nfram && nsl == 1 && bounds[0] == 0 && bounds[1] == h->n_inst;
        if (fused) {
            const EbuK1Args a = {src, stride, nch, (int)pos, h->cf, ck, (float)h->fragm, h->d_z, h->d_frpwr, h->d_fragpw, (int)h->n_inst};
            if (int rc = k1_fused (after_arg, a)) return rc;
        }
        const bool al = aligned && (done % 4 == 0);
        CUtensorMap tmap;
        const bool tma = !fused && !multi && al && h->use_tma && h->nchan <= 2 && !h->weighted && tma_input_map (&tmap, src, stride, (uint32_t)nch, pos);
        for (int sl = 0; !fused && sl < nsl; ++sl) {
            const int kf = (int)(bounds[sl] * h->nchan), ke = (int)(bounds[sl + 1] * h->nchan);
            if (ke <= kf) continue;
            if (ready && done == 0) B200M_CUDA (cudaStreamWaitEvent (st, ready[sl], 0));
            const int cpw = (32 / (int)h->nchan) * (int)h->nchan;          // a warp takes whole instances only
            const int nwarps = (ke - kf + cpw - 1) / cpw;
            dim3 grid ((nwarps + EBU_WARPS - 1) / EBU_WARPS), blk (EBU_WARPS * 32);
            const int pt = (after_k1 && done == 0) ? 1 : 0;
            if (h->weighted)                                     // weighted banks: the run-time channel count, lanes grouped per instance
                ebu_k1w_for (al, multi, d_len)<<<grid, blk, EBU_SMEM_BYTES, st>>> (src, stride, nch, kf, ke, (int)pos, h->cf, ck, (float)h->fragm, h->d_z, h->d_frpwr, h->d_fragpw, (int)h->n_inst, pt, h->gw, d_len);
            else if (h->nchan <= 2 && h->split && !tma && !multi) {       // the opt-in variants know the chunk list only
                dim3 sgrid ((nwarps + EBU_SPLIT_PAIRS - 1) / EBU_SPLIT_PAIRS), sblk (2 * EBU_SPLIT_PAIRS * 32);
                ebu_k1s_for (h->nchan, al)<<<sgrid, sblk, EBU_SPLIT_SMEM, st>>> (src, stride, nch, kf, ke, (int)pos, h->cf, ck, (float)h->fragm, h->d_z, h->d_frpwr, h->d_fragpw, (int)h->n_inst, pt);
            }
            else if (tma) ebu_k1t_for (h->nchan)<<<grid, blk, EBU_TMA_SMEM, st>>> (tmap, nch, kf, ke, (int)pos, h->cf, ck, (float)h->fragm, h->d_z, h->d_frpwr, h->d_fragpw, (int)h->n_inst, pt);
            // 1..5 channels; surround banks (3..5) with the lanes grouped per instance
            else ebu_k1_for (h->nchan, al, multi, d_len)<<<grid, blk, EBU_SMEM_BYTES, st>>> (src, stride, nch, kf, ke, (int)pos, h->cf, ck, (float)h->fragm, h->d_z, h->d_frpwr, h->d_fragpw, (int)h->n_inst, pt, d_len);
            B200M_LAUNCHED (1);
        }
        if (after_k1 && done == 0) { if (int rc = after_k1 (after_arg)) return rc; }      // work to enqueue right behind the first K1
        for (int f = 0; f < nfrag; ++f) {                    // fragments complete in order; each may trigger gating
            ebu_fragment_kernel<<<(h->n_inst + K2A_THREADS - 1) / K2A_THREADS, K2A_THREADS, 0, st>>> (
                (int)h->n_inst, f, ck.fph, h->tmod, h->fragm, (int)nfram, h->d_fragpw, h->d_ring, h->d_ctl, h->d_res, h->d_histM, h->d_histS, h->d_cnt, d_len, h->ring.log);
            B200M_LAUNCHED (1);
            // K2b behind fragment f only if some class completing its fragment f has an integrating member whose S period wraps
            // there: a later addpoint in the same block would otherwise be gated into the statistics
            bool wrap = false;
            int q = 0;
            for (auto& c : h->cls) {
                if (!multi || f < h->nf[q]) wrap |= b200m_ebu::phase_tick (c.second);
                ++q;
            }
            if (d_len) wrap |= h->ragged_tick (f);
            if (wrap) {
                ebu_gate_kernel<<<(h->n_inst + K2B_WARPS - 1) / K2B_WARPS, K2B_WARPS * 32, 0, st>>> (
                    (int)h->n_inst, h->d_ctl, h->d_res, h->d_histM, h->d_histS, h->d_cnt, h->d_binpow, h->ring.log);
                B200M_LAUNCHED (1);
            }
        }
        done += pos;
    }
    if (d_len) {                                             // behind the fragment kernels, which read the clocks the block began with
        ebu_ragged_clock_kernel<<<(h->n_inst + 255) / 256, 256, 0, st>>> ((int)h->n_inst, d_len, (int)nfram, h->fragm, h->d_fph);
        B200M_LAUNCHED (1);
        h->ragged_join (len, nfram);
    }
    h->tmod = (int)((h->tmod + nfram) % (uint32_t)h->fragm);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

static int ebu_process (b200m_ebu* h, const float* d_in, size_t stride, uint32_t nfram, cudaStream_t st, const uint32_t* len = nullptr)
{
    const uint32_t bounds[2] = {0, h->n_inst};
    if (len) if (int rc = h->rag.put (len, h->n_inst, st)) return rc;
    return ebu_process_sliced (h, d_in, stride, nfram, st, 1, bounds, nullptr, nullptr, nullptr, nullptr, len, len ? h->rag.d : nullptr);
}

static int ebu_block (b200m_ebu* h, const float* in, size_t stride, uint32_t nfram, bool host, void* stream, const uint32_t* len)
{
    return bank_call (h, in, stride, nfram, host, stream, h ? (size_t)h->n_inst * h->nchan : 0, h ? h->n_inst : 0, len, no_check,
                      [&] (const float* d_in, size_t ds, cudaStream_t st, const uint32_t* rlen) { return ebu_process (h, d_in, ds, nfram, st, rlen); });
}

int b200m_ebu_process_device (b200m_ebu* h, const float* d_in, size_t stride, uint32_t nfram, void* stream)
{
    return ebu_block (h, d_in, stride, nfram, false, stream, nullptr);
}

int b200m_ebu_process_host (b200m_ebu* h, const float* in, size_t stride, uint32_t nfram)
{
    return ebu_block (h, in, stride, nfram, true, nullptr, nullptr);
}

int b200m_ebu_process_ragged_device (b200m_ebu* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream)
{
    return ebu_block (h, d_in, stride, nfram, false, stream, len);
}

int b200m_ebu_process_ragged_host (b200m_ebu* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len)
{
    return ebu_block (h, in, stride, nfram, true, nullptr, len);
}

int b200m_ebu_results (b200m_ebu* h, b200m_ebu_result* out, void* stream)
{
    if (!h || !out) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->stream (stream);
    B200M_CUDA (cudaMemcpyAsync (out, h->d_res, h->n_inst * sizeof (b200m_ebu_result), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_ebu_log_enable (b200m_ebu* h, uint32_t capacity, void* stream)
{
    return ebu_log_enable (h, capacity, false, stream);
}

uint32_t b200m_ebu_log_capacity (const b200m_ebu* h)
{
    return h ? h->ring.log.cap : 0;
}

int b200m_ebu_log_drain (b200m_ebu* h, b200m_ebu_point* out, uint32_t* count, uint64_t* lost, void* stream)
{
    return ebu_log_drain (h, (float*)out, count, lost, stream, false);
}

int b200m_ebu_histogram (b200m_ebu* h, uint32_t inst, int32_t* hist_M, int32_t* hist_S, void* stream)
{
    if (!h || !hist_M || !hist_S || inst >= h->n_inst) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->stream (stream);
    B200M_CUDA (cudaMemcpyAsync (hist_M, h->d_histM + (size_t)inst * HIST_PITCH, 751 * sizeof (int), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaMemcpyAsync (hist_S, h->d_histS + (size_t)inst * HIST_PITCH, 751 * sizeof (int), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

// ---- snapshot / restore (SURVEY §5: the reference never saves DSP state; a batch engine integrating for hours should) ----
// blob = header (the bank time mod fragm), the host-side phase book-keeping per instance (phase int32, then integ, base, frozen
// and its phase class's fragment counter G as bytes), then every device state array in a fixed order.  The class census is
// rebuilt from the per-instance entries.
namespace {
struct EbuSnapHead { uint32_t magic, n_inst, nchan; float fsamp; int32_t tmod, pad[3]; };
constexpr uint32_t EBU_SNAP_MAGIC = 0x42453032u;              // "BE02": per-instance fragment phases
constexpr uint32_t EBU_SNAP_MAGIC_W = 0x42573032u;            // "BW02": the same for a weighted bank, its EBU_MAXCH_W gains follow the header
constexpr size_t EBU_SNAP_HOST_PER_INST = 8;
size_t ebu_head_bytes (const b200m_ebu* h) { return sizeof (EbuSnapHead) + (h->weighted ? sizeof (h->gw.g) : 0); }
struct EbuSeg { void* p; size_t bytes; };
int ebu_segments (b200m_ebu* h, EbuSeg* seg)
{
    const size_t n = h->n_inst, nch = (size_t)h->n_inst * h->nchan;
    int k = 0;
    seg[k++] = {h->d_z, 4 * nch * sizeof (float)}; seg[k++] = {h->d_frpwr, n * sizeof (float)}; seg[k++] = {h->d_ring, 64 * n * sizeof (float)};
    seg[k++] = {h->d_ctl, n * sizeof (EbuCtl)}; seg[k++] = {h->d_res, n * sizeof (b200m_ebu_result)};
    seg[k++] = {h->d_histM, (size_t)HIST_PITCH * n * sizeof (int)}; seg[k++] = {h->d_histS, (size_t)HIST_PITCH * n * sizeof (int)};
    seg[k++] = {h->d_cnt, 4 * n * sizeof (int)}; seg[k++] = {h->d_fph, n * sizeof (int)};
    return k;
}
}

size_t b200m_ebu_snapshot_size (b200m_ebu* h)
{
    if (!h) return 0;
    EbuSeg seg[9]; const int k = ebu_segments (h, seg);
    size_t b = ebu_head_bytes (h) + EBU_SNAP_HOST_PER_INST * (size_t)h->n_inst;
    b = (b + 15) & ~size_t (15);
    for (int i = 0; i < k; ++i) b += (seg[i].bytes + 15) & ~size_t (15);
    return b;
}

int b200m_ebu_snapshot (b200m_ebu* h, void* buf, size_t bytes, void* stream)
{
    if (!h || !buf || bytes < b200m_ebu_snapshot_size (h)) return set_err (B200M_E_INVAL, "bad argument / buffer too small");
    DeviceGuard g (h->device);
    cudaStream_t st = h->stream (stream);
    uint8_t* o = (uint8_t*)buf;
    EbuSnapHead hd = {h->weighted ? EBU_SNAP_MAGIC_W : EBU_SNAP_MAGIC, h->n_inst, h->nchan, h->fsamp, h->tmod, {0, 0, 0}};
    memcpy (o, &hd, sizeof (hd)); o += sizeof (hd);
    if (h->weighted) { memcpy (o, h->gw.g, sizeof (h->gw.g)); o += sizeof (h->gw.g); }
    const size_t n = h->n_inst;
    memcpy (o, h->ph.data (), 4 * n); o += 4 * n;
    memcpy (o, h->integ.data (), n); o += n; memcpy (o, h->base.data (), n); o += n; memcpy (o, h->frozen.data (), n); o += n;
    for (size_t i = 0; i < n; ++i) *o++ = (uint8_t)h->cls.find (h->ph[i])->second.G;
    o = (uint8_t*)buf + ((ebu_head_bytes (h) + EBU_SNAP_HOST_PER_INST * n + 15) & ~size_t (15));
    EbuSeg seg[9]; const int k = ebu_segments (h, seg);
    for (int i = 0; i < k; ++i) { B200M_CUDA (cudaMemcpyAsync (o, seg[i].p, seg[i].bytes, cudaMemcpyDeviceToHost, st)); o += (seg[i].bytes + 15) & ~size_t (15); }
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_ebu_restore (b200m_ebu* h, const void* buf, size_t bytes, void* stream)
{
    if (!h || !buf || bytes < b200m_ebu_snapshot_size (h)) return set_err (B200M_E_INVAL, "bad argument / buffer too small");
    EbuSnapHead hd; memcpy (&hd, buf, sizeof (hd));
    if (hd.magic != (h->weighted ? EBU_SNAP_MAGIC_W : EBU_SNAP_MAGIC) || hd.n_inst != h->n_inst || hd.nchan != h->nchan || hd.fsamp != h->fsamp)
        return set_err (B200M_E_INVAL, "snapshot does not match this bank (weights / instances / channels / sample rate)");
    if (h->weighted && memcmp ((const uint8_t*)buf + sizeof (hd), h->gw.g, sizeof (h->gw.g)) != 0)
        return set_err (B200M_E_INVAL, "snapshot of a bank with other channel weights");
    DeviceGuard g (h->device);
    cudaStream_t st = h->stream (stream);
    const uint8_t* o = (const uint8_t*)buf + ebu_head_bytes (h);
    const size_t n = h->n_inst;
    h->tmod = hd.tmod;
    memcpy (h->ph.data (), o, 4 * n); o += 4 * n;
    memcpy (h->integ.data (), o, n); o += n; memcpy (h->base.data (), o, n); o += n; memcpy (h->frozen.data (), o, n); o += n;
    h->cls.clear ();
    for (size_t i = 0; i < n; ++i) {
        EbuPhase& c = h->cls[h->ph[i]];
        c.n++; c.G = o[i];
        if (h->integ[i]) c.cnt10[h->base[i]]++;
    }
    o = (const uint8_t*)buf + ((ebu_head_bytes (h) + EBU_SNAP_HOST_PER_INST * n + 15) & ~size_t (15));
    EbuSeg seg[9]; const int k = ebu_segments (h, seg);
    for (int i = 0; i < k; ++i) { B200M_CUDA (cudaMemcpyAsync (seg[i].p, o, seg[i].bytes, cudaMemcpyHostToDevice, st)); o += (seg[i].bytes + 15) & ~size_t (15); }
    // the log's dBTP plane: the open fragments' true-peak maxima belong to the bank before the restore, the snapshot has none
    if (h->tp.open) B200M_CUDA (cudaMemsetAsync (h->tp.open, 0, n * sizeof (float), st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_ebu_coeffs (const b200m_ebu* h, float o[7])
{
    if (!h || !o) return set_err (B200M_E_INVAL, "NULL argument");
    o[0] = h->cf.a0; o[1] = h->cf.a1; o[2] = h->cf.a2; o[3] = h->cf.b1; o[4] = h->cf.b2; o[5] = h->cf.c3; o[6] = h->cf.c4;
    return 0;
}

int b200m_ebu_state (b200m_ebu* h, uint32_t inst, float* z, float* power64, float* frpwr, int32_t c4[4], void* stream)
{
    if (!h || !z || !power64 || !frpwr || !c4 || inst >= h->n_inst) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->stream (stream);
    const size_t nch = (size_t)h->n_inst * h->nchan;
    for (uint32_t c = 0; c < h->nchan; ++c)
        for (int q = 0; q < 4; ++q)
            B200M_CUDA (cudaMemcpyAsync (z + 4 * c + q, h->d_z + q * nch + (size_t)inst * h->nchan + c, sizeof (float), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaMemcpy2DAsync (power64, sizeof (float), h->d_ring + inst, (size_t)h->n_inst * sizeof (float), sizeof (float), 64, cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaMemcpyAsync (frpwr, h->d_frpwr + inst, sizeof (float), cudaMemcpyDeviceToHost, st));
    EbuCtl c;
    B200M_CUDA (cudaMemcpyAsync (&c, h->d_ctl + inst, sizeof (c), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    c4[0] = h->frcnt_of (h->ph[inst]); c4[1] = c.wrind; c4[2] = c.div1; c4[3] = c.div2;
    return 0;
}

int b200m_ebu_mix_reduce (b200m_ebu* h, int32_t* d_out, void* stream)
{
    if (!h || !d_out) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->stream (stream);
    B200M_CUDA (cudaMemsetAsync (d_out, 0, B200M_MIX_WORDS * sizeof (int32_t), st));
    const unsigned slices = (unsigned)std::min<uint32_t> (h->n_inst, 128u);      // ~24 x 128 CTAs: enough loads in flight to stream the histograms
    ebu_mix_reduce_kernel<<<dim3 ((B200M_MIX_WORDS + 63) / 64, slices), 64, 0, st>>> ((int)h->n_inst, h->d_histM, h->d_histS, h->d_cnt, d_out);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

int b200m_ebu_mix_finish (b200m_ebu* h, const int32_t* d_mix, float out5[5], void* stream)
{
    if (!h || !d_mix || !out5) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->stream (stream);
    ebu_mix_finish_kernel<<<1, 32, 0, st>>> (d_mix, h->d_binpow, h->d_out5);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaMemcpyAsync (out5, h->d_out5, 5 * sizeof (float), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_ebu_group_reduce (b200m_ebu* h, const uint32_t* group, uint32_t n_groups, int32_t* d_out, void* stream)
{
    if (!h || !group || !d_out) return set_err (B200M_E_INVAL, "NULL argument");
    if (int rc = group_check (group, h->n_inst, n_groups, B200M_MAX_GROUPS)) return rc;
    DeviceGuard g (h->device);
    cudaStream_t st = h->stream (stream);
    if (int rc = h->grp.assign (group, h->n_inst, n_groups, B200M_MAX_GROUPS, st)) return rc;
    const uint32_t nm = h->grp.members;
    B200M_CUDA (cudaMemsetAsync (d_out, 0, (size_t)n_groups * B200M_MIX_WORDS * sizeof (int32_t), st));
    if (nm) {
        ebu_group_reduce_kernel<<<(nm + GRP_CHUNK - 1) / GRP_CHUNK, GRP_THREADS, 0, st>>> (h->d_histM, h->d_histS, h->d_cnt, h->grp.d_members (),
                                                                                         h->grp.d_album (), (int)nm, d_out);
        B200M_LAUNCHED (1);
    }
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

int b200m_ebu_group_finish (b200m_ebu* h, const int32_t* d_groups, uint32_t n_groups, float* out5, void* stream)
{
    if (!h || !d_groups || !out5) return set_err (B200M_E_INVAL, "NULL argument");
    if (n_groups == 0 || n_groups > B200M_MAX_GROUPS) return set_err (B200M_E_INVAL, "n_groups %u outside 1..%u", n_groups, B200M_MAX_GROUPS);
    DeviceGuard g (h->device);
    cudaStream_t st = h->stream (stream);
    if (n_groups > h->grp5_cap) {                           // the previous call synchronised: nothing in flight uses the old buffer
        cudaFree (h->d_grp5); h->d_grp5 = nullptr; h->grp5_cap = 0;
        if (cudaMalloc ((void**)&h->d_grp5, (size_t)n_groups * 5 * sizeof (float)) != cudaSuccess) {
            cudaGetLastError ();
            return set_err (B200M_E_NOMEM, "album results of %u groups: out of device memory", n_groups);
        }
        h->grp5_cap = n_groups;
    }
    ebu_group_finish_kernel<<<(n_groups + GRP_FIN_WARPS - 1) / GRP_FIN_WARPS, GRP_FIN_WARPS * 32, 0, st>>> ((int)n_groups, d_groups, h->d_binpow, h->d_grp5);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    B200M_CUDA (cudaMemcpyAsync (out5, h->d_grp5, (size_t)n_groups * 5 * sizeof (float), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

}  // extern "C"

int ebu_log_enable (b200m_ebu* h, uint32_t capacity, bool dbtp, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    if (dbtp && capacity && h->fragm < TPLOG_MIN_FRAGM)
        return set_err (B200M_E_UNSUPPORTED, "the dBTP plane needs fragments of >= %d frames (a sample rate of >= %d Hz)", TPLOG_MIN_FRAGM, 20 * TPLOG_MIN_FRAGM);
    DeviceGuard g (h->device);
    cudaStream_t st = h->stream (stream);
    if (h->ring.log.pts) {                                   // kernels in flight may still write the old log
        B200M_CUDA (cudaStreamSynchronize (st));
        h->log_free ();
    }
    if (capacity == 0) return 0;
    const size_t n = h->n_inst;
    cudaError_t e = h->ring.alloc (n, capacity, EBU_LOG_FIELDS + (dbtp ? 1 : 0), st);
    if (dbtp) {
        EbuTpPlane tp = {};
        tp.E = (int)(B200M_MAX_BLOCK / (uint32_t)h->fragm) + 2;
        const size_t fm = (size_t)tp.E * n * h->nchan * sizeof (unsigned);
        if (e == cudaSuccess) e = cudaMalloc ((void**)&tp.fmax, fm);
        h->tp = tp;                                          // log_free releases whatever was allocated
        if (e == cudaSuccess) e = cudaMalloc ((void**)&h->tp.fph0, n * sizeof (int));
        if (e == cudaSuccess) e = cudaMalloc ((void**)&h->tp.open, n * sizeof (float));
        if (e == cudaSuccess) e = cudaMalloc ((void**)&h->tp.filled, n * sizeof (unsigned long long));
        if (e == cudaSuccess) e = cudaMemsetAsync (h->tp.fmax, 0, fm, st);
        if (e == cudaSuccess) e = cudaMemsetAsync (h->tp.open, 0, n * sizeof (float), st);
        if (e == cudaSuccess) e = cudaMemsetAsync (h->tp.filled, 0, n * sizeof (unsigned long long), st);
    }
    if (e != cudaSuccess) {
        h->log_free ();
        cudaGetLastError ();                                 // a failed allocation is not sticky: later calls must not see it
        if (e == cudaErrorMemoryAllocation) return set_err (B200M_E_NOMEM, "loudness log of %u points x %u instances: out of device memory", capacity, h->n_inst);
        return cuda_fail (e, "b200m_ebu_log_enable", __FILE__, __LINE__);
    }
    return 0;
}

int ebu_log_drain (b200m_ebu* h, float* out, uint32_t* count, uint64_t* lost, void* stream, bool dbtp)
{
    if (!h || !out || !count || !lost) return set_err (B200M_E_INVAL, "NULL argument");
    if (!h->ring.log.pts) return set_err (B200M_E_INVAL, "the loudness log is off (b200m_ebu_log_enable)");
    if (dbtp && !h->tp.fmax) return set_err (B200M_E_INVAL, "the loudness log has no dBTP plane (b200m_r128_log_enable)");
    DeviceGuard g (h->device);
    cudaStream_t st = h->stream (stream);
    if (dbtp) return log_drain<EBU_LOG_FIELDS + 1, 32> (h->ring, h->n_inst, out, count, lost, st);
    return log_drain<EBU_LOG_FIELDS, 32> (h->ring, h->n_inst, out, count, lost, st);
}

bool ebu_tp_view (b200m_ebu* h, EbuTpView* v)
{
    if (!h->tp.fmax) return false;
    *v = {h->ring.log, h->tp, h->d_fph, h->tmod, h->fragm};
    return true;
}

RaggedLen& ebu_lens (b200m_ebu* h) { return h->rag; }
void ebu_follow (b200m_ebu* h, const BankPath* owner) { h->owner = owner; }
