// ppm.cu — needle-meter ballistics bank: VU, IEC type I / II peak programme meters, BBC M/S PPM.
//
// Replaces, for N meters at once, LV2M::Vumeterdsp (jmeters/vumeterdsp.cc:45-93), LV2M::Iec1ppmdsp / Iec2ppmdsp
// (jmeters/iec1ppmdsp.cc:47-99, iec2ppmdsp.cc:47-99) and LV2M::Msppmdsp (jmeters/msppmdsp.cc:50-143) as driven by
// run() and bbcm_run() (src/meters.cc:298-331,552-589).  SURVEY.md §8(f) rank 3: the same recurrence family as the
// true-peak ballistics, without the oversampler.  One lane per meter (M/S: one lane per stereo pair, both meters),
// [32 rows x 64 samples] cp.async tiles per warp, four independent warps per CTA; operation order is the reference's,
// unfused, so every state word is bit-identical.
#include <math.h>
#include <stdlib.h>
#include <vector>
#include "common.cuh"

namespace b200m {

constexpr int PPM_T = 64, PPM_P = PPM_T + 4, PPM_STAGES = 3, PPM_WARPS = 4;
constexpr int PPM_PLANE = 32 * PPM_P;                      // floats of one [32 x 64] plane

struct PpmParams { float w1, w2, w3; };

constexpr int PPM_EDGES = B200M_PPM_HIST_BINS - 1;

// the needle histogram plane (b200m_ppm_hist_enable), one allocation: counts, then stats, then the edge table
struct PpmHist {
    unsigned long long* cnt;                               // [n_meters][B200M_PPM_HIST_BINS]
    b200m_ppm_hist_stats* st;                              // [n_meters]
    const float* edges;                                    // [PPM_EDGES]
    float lim;                                             // L
};

// KIND 0: VU   1: IEC I/II PPM   3: M/S PPM (two planes: L and R rows of the pair)
// RAG (b200m_ppm_process_ragged_*): unit u runs process() over its first rlen[u] <= nfram frames only.  Its lane stops at its own
// (rlen[u] / 4) * 4; the warp still stages whole [32 x 64] tiles up to its longest row, so frames past a row's end are loaded but never
// reach its filters.  A unit with rlen[u] == 0 was not called: no clamp, scrub or _res store.
// HIST (b200m_ppm_hist_enable): after each group of 4 frames every meter forms the reading v = g * s of the needle value s the
// reference compares with m, and counts it (include/b200meters.h).  The needle moves slowly against the 0.5 dB bins, so a lane holds
// each meter's (bin, run) with the bin's two edges in registers and adds the run to the meter's own row with one fire-and-forget
// atomic (RED) only when the bin changes and at kernel end; the edge table sits in shared memory for the search.  The meter's
// statistics are loaded at kernel start and stored at kernel end: the lane owns its meters.  The recurrences, states and ports are
// the same bits as without the plane.
template <int KIND, bool ALIGNED, bool RAG = false, bool HIST = false>
__global__ void __launch_bounds__ (PPM_WARPS * 32)
ppm_kernel (const float* __restrict__ in, size_t stride, int n_units, int nfram, PpmParams pr, const float2* __restrict__ mv /* M/S: [unit] {mv_m, mv_s} */,
            float* __restrict__ z1s, float* __restrict__ z2s, float* __restrict__ ms, int* __restrict__ ress, const uint32_t* __restrict__ rlen,
            float gr /* read()'s _g */, PpmHist hp)
{
    constexpr int PLANES = KIND == 3 ? 2 : 1;
    extern __shared__ __align__ (16) float ppm_smem[];
    const float* E = nullptr;                              // HIST: the edge table
    if constexpr (HIST) {
        __shared__ float ppm_edges[PPM_EDGES];
        for (int i = threadIdx.x; i < PPM_EDGES; i += blockDim.x) ppm_edges[i] = hp.edges[i];
        __syncthreads ();                                  // before any warp leaves
        E = ppm_edges;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int u0 = (blockIdx.x * PPM_WARPS + warp) * 32;    // first unit (meter, or stereo pair) of this warp
    if (u0 >= n_units) return;
    float* ring = ppm_smem + warp * (PPM_STAGES * PLANES * PPM_PLANE);
    const int u = min (u0 + lane, n_units - 1);
    const bool live = (u0 + lane) < n_units;
    int nproc = (nfram / 4) * 4;                           // "n /= 4": the last n mod 4 samples are ignored
    int rl = nfram, lproc = nproc;                         // RAG: this lane's length and its processed samples
    if constexpr (RAG) {
        rl = (int)rlen[u]; lproc = (rl / 4) * 4;
        nproc = __reduce_max_sync (0xffffffffu, lproc);    // the warp stages up to its longest row
    }
    const int ntiles = (nproc + PPM_T - 1) / PPM_T;

    auto issue = [&] (int t) {
        if (t < ntiles) {
            float* dst = ring + (t % PPM_STAGES) * (PLANES * PPM_PLANE);
            const int s0 = t * PPM_T;
#pragma unroll
            for (int pl = 0; pl < PLANES; ++pl) {
                if (ALIGNED) {
                    const int c4 = (lane & 15) * 4;
                    const int left = (nproc - (s0 + c4)) * 4;
                    const int nb = left >= 16 ? 16 : (left > 0 ? left : 0);
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const int r = 2 * i + (lane >> 4);
                        const int ur = min (u0 + r, n_units - 1);
                        const float* src = in + (size_t)(PLANES * ur + pl) * stride + s0 + c4;
                        cp_async16 (dst + pl * PPM_PLANE + r * PPM_P + c4, nb ? src : in, nb);
                    }
                } else {
#pragma unroll 4
                    for (int r = 0; r < 32; ++r) {
                        const int ur = min (u0 + r, n_units - 1);
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int c = lane + 32 * h;
                            const bool ok = (s0 + c) < nproc;
                            cp_async4 (dst + pl * PPM_PLANE + r * PPM_P + c, ok ? in + (size_t)(PLANES * ur + pl) * stride + s0 + c : in, ok ? 4 : 0);
                        }
                    }
                }
            }
        }
        cp_async_commit ();
    };

    // meter state: for M/S the pair's two meters sit at 2u (mid) and 2u + 1 (side)
    constexpr int NM = KIND == 3 ? 2 : 1;
    float z1[NM], z2[NM], m[NM];
#pragma unroll
    for (int q = 0; q < NM; ++q) {
        const int idx = NM * u + q;
        const float a = z1s[idx], b = z2s[idx];
        if (KIND == 0) { z1[q] = a > 20 ? 20 : (a < -20 ? -20 : a); z2[q] = b > 20 ? 20 : (b < -20 ? -20 : b); }   // vumeterdsp.cc:49-50
        else           { z1[q] = a > 20 ? 20 : (a < 0 ? 0 : a);     z2[q] = b > 20 ? 20 : (b < 0 ? 0 : b); }         // iec1ppmdsp.cc:51-52
        m[q] = ress[idx] ? 0.0f : ms[idx];
    }
    const float w4 = __fmul_rn (4.0f, pr.w1);
    const float2 g = KIND == 3 ? mv[u] : make_float2 (1.0f, 1.0f);

    // HIST, per meter: the open run hr of readings in bin hb, whose edges are [hlo, hhi), and the statistics of b200m_ppm_hist_stats
    int hb[NM] = {}; uint32_t hr[NM] = {}; float hlo[NM] = {}, hhi[NM] = {}, pk[NM] = {};
    unsigned long long nnf[NM] = {}, nov[NM] = {}, novs[NM] = {}, nlong[NM] = {}, nrun[NM] = {};
    if constexpr (HIST) {
#pragma unroll
        for (int q = 0; q < NM; ++q) {
            const b200m_ppm_hist_stats& a = hp.st[NM * u + q];
            nnf[q] = a.nonfinite; nov[q] = a.over_groups; novs[q] = a.overs; nlong[q] = a.longest_over; nrun[q] = a.run; pk[q] = a.peak;
            hlo[q] = INFINITY; hhi[q] = -INFINITY;         // an empty range: the first reading searches
        }
    }
    auto flush = [&] (int q) {                             // lanes past the bank repeat its last unit: they add nothing
        if (live && hr[q]) atomicAdd (hp.cnt + (size_t)(NM * u + q) * B200M_PPM_HIST_BINS + hb[q], (unsigned long long)hr[q]);
    };
    auto tally = [&] (int q, float s) {
        const float v = __fmul_rn (gr, s);
        if (!finitef_ (v)) { ++nnf[q]; return; }           // no bin, and the over run stands
        if (v > pk[q]) pk[q] = v;
        if (v >= hp.lim) { ++nov[q]; novs[q] += nrun[q] == 0; ++nrun[q]; if (nrun[q] > nlong[q]) nlong[q] = nrun[q]; }
        else nrun[q] = 0;
        if (v >= hlo[q] && v < hhi[q]) { ++hr[q]; return; }
        flush (q);
        // bin = #{k : v >= E[k]}: an estimate from 40 log10 v + 161, corrected against the table, which alone defines the bins
        int k = 0;
        if (v >= E[0]) {
            k = (int)fminf (fmaxf (__fadd_rn (__fmul_rn (__log2f (v), 12.0411998f), 161.0f), 1.0f), (float)PPM_EDGES);
            while (k > 1 && v < E[k - 1]) --k;
            while (k < PPM_EDGES && v >= E[k]) ++k;
        }
        hb[q] = k; hr[q] = 1;
        hlo[q] = k > 0 ? E[k - 1] : -INFINITY; hhi[q] = k < PPM_EDGES ? E[k] : INFINITY;
    };

    auto group = [&] (const float4 a, const float4 b) {
        const float xa[4] = {a.x, a.y, a.z, a.w}, xb[4] = {b.x, b.y, b.z, b.w};
        if (KIND == 0) {                                   // vumeterdsp.cc:57-68
            const float t2 = __fmul_rn (z2[0], 0.5f);      // z2 / 2 (exact either way)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float t1 = __fsub_rn (fabsf (xa[i]), t2);
                z1[0] = __fadd_rn (z1[0], __fmul_rn (pr.w1, __fsub_rn (t1, z1[0])));
            }
            z2[0] = __fadd_rn (z2[0], __fmul_rn (w4, __fsub_rn (z1[0], z2[0])));
            if (z2[0] > m[0]) m[0] = z2[0];
            if constexpr (HIST) tally (0, z2[0]);
        } else {
#pragma unroll
            for (int q = 0; q < NM; ++q) { z1[q] = __fmul_rn (z1[q], pr.w3); z2[q] = __fmul_rn (z2[q], pr.w3); }   // iec1ppmdsp.cc:59-60
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float t[NM];
                if (KIND == 1) t[0] = fabsf (xa[i]);
                else { t[0] = __fmul_rn (g.x, fabsf (__fadd_rn (xa[i], xb[i])));             // msppmdsp.cc:63,97
                       t[NM - 1] = __fmul_rn (g.y, fabsf (__fsub_rn (xa[i], xb[i]))); }
#pragma unroll
                for (int q = 0; q < NM; ++q) {
                    if (t[q] > z1[q]) z1[q] = __fadd_rn (z1[q], __fmul_rn (pr.w1, __fsub_rn (t[q], z1[q])));
                    if (t[q] > z2[q]) z2[q] = __fadd_rn (z2[q], __fmul_rn (pr.w2, __fsub_rn (t[q], z2[q])));
                }
            }
#pragma unroll
            for (int q = 0; q < NM; ++q) {
                const float s = __fadd_rn (z1[q], z2[q]);
                if (s > m[q]) m[q] = s;
                if constexpr (HIST) tally (q, s);
            }
        }
    };

#pragma unroll
    for (int t = 0; t < PPM_STAGES - 1; ++t) issue (t);
    for (int t = 0; t < ntiles; ++t) {
        cp_async_wait<PPM_STAGES - 2> ();
        __syncwarp ();
        const float* base = ring + (t % PPM_STAGES) * (PLANES * PPM_PLANE) + lane * PPM_P;
        const float4* pa = reinterpret_cast<const float4*> (base);
        const float4* pb = reinterpret_cast<const float4*> (base + (PLANES - 1) * PPM_PLANE);
        int ng = (min (PPM_T, nproc - t * PPM_T)) / 4;
        if constexpr (RAG) ng = max (0, min (PPM_T, lproc - t * PPM_T)) / 4;
        for (int q = 0; q < ng; ++q) group (pa[q], pb[q]);
        __syncwarp ();
        issue (t + PPM_STAGES - 1);
    }
    cp_async_wait<0> ();
    if constexpr (HIST) {
#pragma unroll
        for (int q = 0; q < NM; ++q) {
            flush (q);
            if (live) {
                b200m_ppm_hist_stats& a = hp.st[NM * u + q];
                a.nonfinite = nnf[q]; a.over_groups = nov[q]; a.overs = novs[q]; a.longest_over = nlong[q]; a.run = nrun[q]; a.peak = pk[q];
            }
        }
    }
    bool ran = live;                                       // RAG: a unit with length 0 was not called
    if constexpr (RAG) ran = live && rl > 0;
    if (ran) {
#pragma unroll
        for (int q = 0; q < NM; ++q) {
            const int idx = NM * u + q;
            if (KIND == 0) {                               // vumeterdsp.cc:70-72
                if (!finitef_ (z1[q])) { z1s[idx] = 0; m[q] = INFINITY; } else z1s[idx] = z1[q];
                if (!finitef_ (z2[q])) { z2s[idx] = 0; m[q] = INFINITY; } else z2s[idx] = __fadd_rn (z2[q], 1e-10f);
            } else {                                       // iec1ppmdsp.cc:77-78
                z1s[idx] = __fadd_rn (z1[q], 1e-10f); z2s[idx] = __fadd_rn (z2[q], 1e-10f);
            }
            ms[idx] = m[q]; ress[idx] = 0;
        }
    }
}

// RAG: after a ragged block, meter i belongs to unit i / per; a unit with rlen 0 was not called, so it is not read either
template <bool RAG = false>
__global__ void ppm_read_kernel (int nm, float g, const float* __restrict__ ms, int* __restrict__ ress, float* __restrict__ out,
                                 const uint32_t* __restrict__ rlen, int per)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nm) return;
    if (RAG && rlen[(unsigned)i / (unsigned)per] == 0) return;
    out[i] = __fmul_rn (g, ms[i]);                          // read(): _res = true; return _g * _m
    ress[i] = 1;
}
__global__ void ppm_init_kernel (int nm, int* ress) { const int i = blockIdx.x * blockDim.x + threadIdx.x; if (i < nm) ress[i] = 1; }
// meters [m0, m0 + nm) back to a newly constructed meter: z1 z2 m = 0, _res (true), no reading yet
__global__ void ppm_clear_kernel (int m0, int nm, float* z1s, float* z2s, float* ms, float* out, int* ress)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nm) return;
    z1s[m0 + i] = 0; z2s[m0 + i] = 0; ms[m0 + i] = 0; out[m0 + i] = 0; ress[m0 + i] = 1;
}

// the histogram rows of meters [m0, m0 + nm) back to an empty plane: counts and statistics zero, peak -INFINITY
__global__ void ppm_hist_clear_kernel (int m0, int nm, unsigned long long* __restrict__ cnt, b200m_ppm_hist_stats* __restrict__ st)
{
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < (size_t)nm * B200M_PPM_HIST_BINS) cnt[(size_t)m0 * B200M_PPM_HIST_BINS + i] = 0;
    if (i < (size_t)nm) st[m0 + i] = b200m_ppm_hist_stats {0, 0, 0, 0, 0, -INFINITY, 0};
}

}  // namespace b200m

using namespace b200m;

struct b200m_ppm {
    int device, kind; uint32_t n_units, n_meters; float fsamp, g;
    PpmParams pr;
    std::vector<float2> db, mv;                           // M/S: per unit {M, S} gain in dB and as Msppmdsp::_mv; mv is d_mv's host copy
    float2* d_mv = nullptr; bool mv_dirty = false;        // d_mv is rewritten by the next process call
    float *d_z1 = nullptr, *d_z2 = nullptr, *d_m = nullptr, *d_out = nullptr; int* d_res = nullptr;
    RaggedLen rag; bool rag_read = false;                 // ragged blocks: lengths per unit; the last block was ragged (read skips length 0)
    BankPath path;
    // the needle histogram plane (b200m_ppm_hist_enable): [n_meters][242] uint64 counts, then [n_meters] statistics, then the edge
    // table, in one allocation so that a read is one copy; allocated on first use, kept until destroy
    void* d_hist = nullptr;
    bool hist = false;
    float hist_lim = 0.0f;                                // L
    unsigned long long* hist_cnt () const { return (unsigned long long*)d_hist; }
    b200m_ppm_hist_stats* hist_st () const { return (b200m_ppm_hist_stats*)(hist_cnt () + (size_t)n_meters * B200M_PPM_HIST_BINS); }
    float* hist_edges () const { return (float*)(hist_st () + n_meters); }
    size_t hist_read_bytes () const { return (size_t)n_meters * (B200M_PPM_HIST_BINS * sizeof (uint64_t) + sizeof (b200m_ppm_hist_stats)); }
};

// the bin edges e[k] = (float) 10^((-80 + 0.5 k) / 20), computed in double once
static const float* ppm_hist_table ()
{
    static const std::vector<float> e = [] {
        std::vector<float> t (PPM_EDGES);
        for (int k = 0; k < PPM_EDGES; ++k) t[k] = (float)pow (10.0, (-80.0 + 0.5 * k) / 20.0);
        return t;
    } ();
    return e.data ();
}

static void ppm_design (int kind, float fs, float w[4])
{
    if (kind == B200M_PPM_VU)        { w[0] = 11.1f / fs; w[1] = 0; w[2] = 0; w[3] = 1.5f * 1.571f; }                                  // vumeterdsp.cc:89-93
    else if (kind == B200M_PPM_IEC1) { w[0] = 450.0f / fs; w[1] = 1300.0f / fs; w[2] = 1.0f - 5.4f / fs; w[3] = 0.5108f; }            // iec1ppmdsp.cc:93-99
    else                             { w[0] = 200.0f / fs; w[1] = 860.0f / fs;  w[2] = 1.0f - 4.0f / fs; w[3] = 0.5141f; }            // iec2ppmdsp.cc:93-99, msppmdsp.cc:127-133
}

// ppm_kernel of a meter kind (both IEC kinds run KIND 1), an aligned block, a ragged one and the histogram plane
static auto ppm_kernel_for (int kind, bool al, bool rag, bool hist)
{
    return with_int<B200M_PPM_VU, B200M_PPM_MS, 1> (kind, [&] (auto K) {
        return with_bools ([&] (auto AL, auto RAG, auto HIST) { return ppm_kernel<K, AL, RAG, HIST>; }, al, rag, hist);
    });
}

// len (host, every entry <= nfram, some != nfram: ragged_check): unit u runs over its first len[u] frames; nullptr: every unit nfram
static int ppm_process (b200m_ppm* h, const float* d_in, size_t stride, uint32_t nfram, cudaStream_t st, const uint32_t* len = nullptr)
{
    h->rag_read = len != nullptr;
    if (len) if (int rc = h->rag.put (len, h->n_units, st)) return rc;
    if (h->mv_dirty) {
        B200M_CUDA (cudaMemcpyAsync (h->d_mv, h->mv.data (), h->n_units * sizeof (float2), cudaMemcpyHostToDevice, st));
        h->mv_dirty = false;
    }
    const bool al = ((uintptr_t)d_in % 16 == 0) && (stride % 4 == 0);
    const int planes = h->kind == B200M_PPM_MS ? 2 : 1;
    const size_t smem = (size_t)PPM_WARPS * PPM_STAGES * planes * PPM_PLANE * sizeof (float);
    const int nwarps = (h->n_units + 31) / 32;
    dim3 grid ((nwarps + PPM_WARPS - 1) / PPM_WARPS), blk (PPM_WARPS * 32);
    const PpmHist hp = h->hist ? PpmHist {h->hist_cnt (), h->hist_st (), h->hist_edges (), h->hist_lim} : PpmHist {};
    ppm_kernel_for (h->kind, al, len, h->hist)<<<grid, blk, smem, st>>> (d_in, stride, (int)h->n_units, (int)nfram, h->pr, h->d_mv, h->d_z1, h->d_z2,
                                                                     h->d_m, h->d_res, len ? h->rag.d : nullptr, h->g, hp);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

static int ppm_hist_clear (b200m_ppm* h, int m0, int nm, cudaStream_t st)
{
    const size_t n = (size_t)nm * B200M_PPM_HIST_BINS;
    ppm_hist_clear_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>> (m0, nm, h->hist_cnt (), h->hist_st ());
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

extern "C" {

int b200m_design_ppm (int kind, float fsamp, float w[4])
{
    if (!w || kind < 0 || kind > 3 || !(fsamp >= 1000.0f)) return set_err (B200M_E_INVAL, "bad argument");
    ppm_design (kind, fsamp, w);
    return 0;
}

int b200m_ppm_create (b200m_ppm** out, int device, uint32_t n_units, float fsamp, int kind)
{
    if (!out) return set_err (B200M_E_INVAL, "NULL out pointer");
    *out = nullptr;
    if (n_units == 0 || !(fsamp >= 1000.0f) || kind < 0 || kind > 3) return set_err (B200M_E_INVAL, "bad n/fsamp/kind");
    if (b200m_device_count () <= 0) return set_err (B200M_E_NODEVICE, "no CUDA device: b200meters has no CPU path");
    DeviceGuard g (device);
    if (!g.ok) return set_err (B200M_E_NODEVICE, "cannot select CUDA device %d", device);
    b200m_ppm* h = new (std::nothrow) b200m_ppm;
    if (!h) return set_err (B200M_E_NOMEM, "host allocation failed");
    h->device = device; h->kind = kind; h->n_units = n_units; h->n_meters = kind == B200M_PPM_MS ? 2 * n_units : n_units; h->fsamp = fsamp;
    float w[4]; ppm_design (kind, fsamp, w);
    h->pr.w1 = w[0]; h->pr.w2 = w[1]; h->pr.w3 = w[2]; h->g = w[3];
    if (kind == B200M_PPM_MS) {
        h->db.assign (n_units, make_float2 (0, 0)); h->mv.assign (n_units, make_float2 (1, 1));
        b200m_ppm_set_gain (h, -6, -6);                                  // new Msppmdsp (-6) x2, src/meters.cc:210-212
    }
    cudaError_t e = cudaSuccess;
    auto A = [&] (void** p, size_t bytes) { if (e == cudaSuccess) { e = cudaMalloc (p, bytes); if (e == cudaSuccess) e = cudaMemset (*p, 0, bytes); } };
    const size_t nm = h->n_meters;
    A ((void**)&h->d_z1, nm * 4); A ((void**)&h->d_z2, nm * 4); A ((void**)&h->d_m, nm * 4); A ((void**)&h->d_out, nm * 4); A ((void**)&h->d_res, nm * 4);
    if (kind == B200M_PPM_MS) A ((void**)&h->d_mv, n_units * sizeof (float2));
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags (&h->path.own, cudaStreamNonBlocking);
    const int smem_max = PPM_WARPS * PPM_STAGES * 2 * PPM_PLANE * (int)sizeof (float);
    for (int k = B200M_PPM_VU; k <= B200M_PPM_MS; ++k)
        for (const bool al : {false, true})
            for (const bool rag : {false, true})
                for (const bool hist : {false, true})
                    if (e == cudaSuccess) e = cudaFuncSetAttribute (ppm_kernel_for (k, al, rag, hist), cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
    if (e == cudaSuccess) {
        ppm_init_kernel<<<(unsigned)((nm + 255) / 256), 256>>> ((int)nm, h->d_res);    // constructors: _res (true)
        B200M_LAUNCHED (1);
        e = cudaDeviceSynchronize ();
    }
    if (e != cudaSuccess) { int rc = cuda_fail (e, "ppm_create", __FILE__, __LINE__); b200m_ppm_destroy (h); return rc; }
    *out = h;
    return 0;
}

int b200m_ppm_destroy (b200m_ppm* h)
{
    if (!h) return 0;
    DeviceGuard g (h->device);
    cudaDeviceSynchronize ();
    cudaFree (h->d_z1); cudaFree (h->d_z2); cudaFree (h->d_m); cudaFree (h->d_out); cudaFree (h->d_res); cudaFree (h->d_mv); cudaFree (h->d_hist); h->rag.release (); h->path.release ();
    delete h;
    return 0;
}

int b200m_ppm_set_gain_inst (b200m_ppm* h, int32_t unit, float db_m, float db_s)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    if (h->kind != B200M_PPM_MS) return set_err (B200M_E_INVAL, "set_gain applies to the M/S PPM bank");
    if (unit < -1 || unit >= (int32_t)h->n_units) return set_err (B200M_E_INVAL, "bad unit");
    const uint32_t u0 = unit < 0 ? 0 : (uint32_t)unit, u1 = unit < 0 ? h->n_units : u0 + 1;
    for (uint32_t u = u0; u < u1; ++u) {
        // Msppmdsp::set_gain (msppmdsp.cc:135-143): _mv = powf (10, .05 * db), skipped when db is unchanged
        float2& d = h->db[u]; float2& v = h->mv[u];
        if (d.x != db_m) { d.x = db_m; v.x = powf (10, .05 * db_m); h->mv_dirty = true; }
        if (d.y != db_s) { d.y = db_s; v.y = powf (10, .05 * db_s); h->mv_dirty = true; }
    }
    return 0;
}

int b200m_ppm_set_gain (b200m_ppm* h, float db_m, float db_s) { return b200m_ppm_set_gain_inst (h, -1, db_m, db_s); }

int b200m_ppm_clear (b200m_ppm* h, int32_t unit, void* stream)
{
    if (!h || unit < -1 || unit >= (int32_t)h->n_units) return set_err (B200M_E_INVAL, "bad argument");
    DeviceGuard g (h->device);
    const int per = h->kind == B200M_PPM_MS ? 2 : 1;
    const int m0 = unit < 0 ? 0 : per * unit, nm = unit < 0 ? (int)h->n_meters : per;
    cudaStream_t st = h->path.stream (stream);
    ppm_clear_kernel<<<(nm + 255) / 256, 256, 0, st>>> (m0, nm, h->d_z1, h->d_z2, h->d_m, h->d_out, h->d_res);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    if (h->hist)                                           // a cleared unit is a fresh meter for the histogram too
        if (int rc = ppm_hist_clear (h, m0, nm, st)) return rc;
    if (h->kind == B200M_PPM_MS) {                         // the constructor's gains: a fresh Msppmdsp (-6) pair
        const uint32_t u0 = unit < 0 ? 0 : (uint32_t)unit, u1 = unit < 0 ? h->n_units : u0 + 1;
        for (uint32_t u = u0; u < u1; ++u) { h->db[u] = make_float2 (0, 0); h->mv[u] = make_float2 (1, 1); }
        return b200m_ppm_set_gain_inst (h, unit, -6, -6);
    }
    return 0;
}

static int ppm_block (b200m_ppm* h, const float* in, size_t stride, uint32_t nfram, bool host, void* stream, const uint32_t* len)
{
    return bank_call (h, in, stride, nfram, host, stream, h ? h->n_meters : 0, h ? h->n_units : 0, len, no_check,
                      [&] (const float* d_in, size_t ds, cudaStream_t st, const uint32_t* rlen) { return ppm_process (h, d_in, ds, nfram, st, rlen); });
}

int b200m_ppm_process_device (b200m_ppm* h, const float* d_in, size_t stride, uint32_t nfram, void* stream)
{
    return ppm_block (h, d_in, stride, nfram, false, stream, nullptr);
}

int b200m_ppm_process_host (b200m_ppm* h, const float* in, size_t stride, uint32_t nfram)
{
    return ppm_block (h, in, stride, nfram, true, nullptr, nullptr);
}

int b200m_ppm_process_ragged_device (b200m_ppm* h, const float* d_in, size_t stride, uint32_t nfram, const uint32_t* len, void* stream)
{
    return ppm_block (h, d_in, stride, nfram, false, stream, len);
}

int b200m_ppm_process_ragged_host (b200m_ppm* h, const float* in, size_t stride, uint32_t nfram, const uint32_t* len)
{
    return ppm_block (h, in, stride, nfram, true, nullptr, len);
}

int b200m_ppm_read_device (b200m_ppm* h, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    DeviceGuard g (h->device);
    const unsigned grid = (h->n_meters + 255) / 256;
    if (h->rag_read)                                      // after a ragged block: units with length 0 were not called
        ppm_read_kernel<true><<<grid, 256, 0, h->path.stream (stream)>>> ((int)h->n_meters, h->g, h->d_m, h->d_res, h->d_out, h->rag.d,
                                                                          h->kind == B200M_PPM_MS ? 2 : 1);
    else ppm_read_kernel<<<grid, 256, 0, h->path.stream (stream)>>> ((int)h->n_meters, h->g, h->d_m, h->d_res, h->d_out, nullptr, 1);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

int b200m_ppm_results (b200m_ppm* h, float* out, void* stream)
{
    if (!h || !out) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    B200M_CUDA (cudaMemcpyAsync (out, h->d_out, h->n_meters * sizeof (float), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_ppm_state (b200m_ppm* h, float* state4, void* stream)
{
    if (!h || !state4) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    const size_t nm = h->n_meters;
    float* tmp = (float*)malloc (4 * nm * sizeof (float));
    if (!tmp) return set_err (B200M_E_NOMEM, "host allocation failed");
    const void* src[4] = {h->d_z1, h->d_z2, h->d_m, h->d_res};
    cudaError_t e = cudaSuccess;
    for (int q = 0; q < 4 && e == cudaSuccess; ++q) e = cudaMemcpyAsync (tmp + q * nm, src[q], nm * 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize (st);
    if (e != cudaSuccess) { free (tmp); return cuda_fail (e, "ppm_state", __FILE__, __LINE__); }
    for (size_t i = 0; i < nm; ++i) {
        state4[4 * i] = tmp[i]; state4[4 * i + 1] = tmp[nm + i]; state4[4 * i + 2] = tmp[2 * nm + i];
        state4[4 * i + 3] = (float)((const int*)(tmp + 3 * nm))[i];
    }
    free (tmp);
    return 0;
}

int b200m_ppm_hist_enable (b200m_ppm* h, int enable, float limit_db, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    if (isnan (limit_db)) return set_err (B200M_E_INVAL, "limit_db must not be NaN");
    DeviceGuard g (h->device);
    if (!enable) { h->hist = false; return 0; }           // the plane's memory stays for the next enable
    cudaStream_t st = h->path.stream (stream);
    if (!h->d_hist) {
        const cudaError_t e = cudaMalloc (&h->d_hist, h->hist_read_bytes () + PPM_EDGES * sizeof (float));
        if (e != cudaSuccess) {
            cudaGetLastError ();                               // a failed allocation is not sticky: later calls must not see it
            h->d_hist = nullptr;
            if (e == cudaErrorMemoryAllocation) return set_err (B200M_E_NOMEM, "needle histogram of %u meters: out of device memory", h->n_meters);
            return cuda_fail (e, "b200m_ppm_hist_enable", __FILE__, __LINE__);
        }
        B200M_CUDA (cudaMemcpyAsync (h->hist_edges (), ppm_hist_table (), PPM_EDGES * sizeof (float), cudaMemcpyHostToDevice, st));
    }
    if (int rc = ppm_hist_clear (h, 0, (int)h->n_meters, st)) return rc;
    h->hist_lim = (float)pow (10.0, (double)limit_db / 20.0);     // +inf dB: no reading is over; -inf dB: L = 0
    h->hist = true;
    return 0;
}

int b200m_ppm_hist_read (b200m_ppm* h, uint64_t* counts, b200m_ppm_hist_stats* stats, void* stream)
{
    if (!h || !counts || !stats) return set_err (B200M_E_INVAL, "NULL argument");
    if (!h->hist) return set_err (B200M_E_INVAL, "the needle histogram plane is off (b200m_ppm_hist_enable)");
    DeviceGuard g (h->device);
    cudaStream_t st = h->path.stream (stream);
    std::vector<unsigned char> buf (h->hist_read_bytes ());
    B200M_CUDA (cudaMemcpyAsync (buf.data (), h->d_hist, buf.size (), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    const size_t nc = (size_t)h->n_meters * B200M_PPM_HIST_BINS * sizeof (uint64_t);
    memcpy (counts, buf.data (), nc);
    memcpy (stats, buf.data () + nc, (size_t)h->n_meters * sizeof (b200m_ppm_hist_stats));
    return 0;
}

int b200m_ppm_hist_edges (float* edges)
{
    if (!edges) return set_err (B200M_E_INVAL, "NULL argument");
    memcpy (edges, ppm_hist_table (), PPM_EDGES * sizeof (float));
    return 0;
}

}  // extern "C"
