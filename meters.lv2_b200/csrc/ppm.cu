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

// KIND 0: VU   1: IEC I/II PPM   3: M/S PPM (two planes: L and R rows of the pair)
template <int KIND, bool ALIGNED>
__global__ void __launch_bounds__ (PPM_WARPS * 32)
ppm_kernel (const float* __restrict__ in, size_t stride, int n_units, int nfram, PpmParams pr, const float2* __restrict__ mv /* M/S: [unit] {mv_m, mv_s} */,
            float* __restrict__ z1s, float* __restrict__ z2s, float* __restrict__ ms, int* __restrict__ ress)
{
    constexpr int PLANES = KIND == 3 ? 2 : 1;
    extern __shared__ __align__ (16) float ppm_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int u0 = (blockIdx.x * PPM_WARPS + warp) * 32;    // first unit (meter, or stereo pair) of this warp
    if (u0 >= n_units) return;
    float* ring = ppm_smem + warp * (PPM_STAGES * PLANES * PPM_PLANE);
    const int u = min (u0 + lane, n_units - 1);
    const bool live = (u0 + lane) < n_units;
    const int nproc = (nfram / 4) * 4;                     // "n /= 4": the last n mod 4 samples are ignored
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
            for (int q = 0; q < NM; ++q) { const float s = __fadd_rn (z1[q], z2[q]); if (s > m[q]) m[q] = s; }
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
        const int ng = (min (PPM_T, nproc - t * PPM_T)) / 4;
        for (int q = 0; q < ng; ++q) group (pa[q], pb[q]);
        __syncwarp ();
        issue (t + PPM_STAGES - 1);
    }
    cp_async_wait<0> ();
    if (live) {
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

__global__ void ppm_read_kernel (int nm, float g, const float* __restrict__ ms, int* __restrict__ ress, float* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nm) return;
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

}  // namespace b200m

using namespace b200m;

struct b200m_ppm {
    int device, kind; uint32_t n_units, n_meters; float fsamp, g;
    PpmParams pr;
    std::vector<float2> db, mv;                           // M/S: per unit {M, S} gain in dB and as Msppmdsp::_mv; mv is d_mv's host copy
    float2* d_mv = nullptr; bool mv_dirty = false;        // d_mv is rewritten by the next process call
    float *d_z1 = nullptr, *d_z2 = nullptr, *d_m = nullptr, *d_out = nullptr; int* d_res = nullptr;
    cudaStream_t own = nullptr; HostStage stage; bool last_host = false;
};

static void ppm_design (int kind, float fs, float w[4])
{
    if (kind == B200M_PPM_VU)        { w[0] = 11.1f / fs; w[1] = 0; w[2] = 0; w[3] = 1.5f * 1.571f; }                                  // vumeterdsp.cc:89-93
    else if (kind == B200M_PPM_IEC1) { w[0] = 450.0f / fs; w[1] = 1300.0f / fs; w[2] = 1.0f - 5.4f / fs; w[3] = 0.5108f; }            // iec1ppmdsp.cc:93-99
    else                             { w[0] = 200.0f / fs; w[1] = 860.0f / fs;  w[2] = 1.0f - 4.0f / fs; w[3] = 0.5141f; }            // iec2ppmdsp.cc:93-99, msppmdsp.cc:127-133
}

static cudaStream_t ppm_stream (b200m_ppm* h, void* stream) { return h->last_host ? h->own : (cudaStream_t)stream; }

static int ppm_process (b200m_ppm* h, const float* d_in, size_t stride, uint32_t nfram, cudaStream_t st)
{
    if (h->mv_dirty) {
        B200M_CUDA (cudaMemcpyAsync (h->d_mv, h->mv.data (), h->n_units * sizeof (float2), cudaMemcpyHostToDevice, st));
        h->mv_dirty = false;
    }
    const bool al = ((uintptr_t)d_in % 16 == 0) && (stride % 4 == 0);
    const int planes = h->kind == B200M_PPM_MS ? 2 : 1;
    const size_t smem = (size_t)PPM_WARPS * PPM_STAGES * planes * PPM_PLANE * sizeof (float);
    const int nwarps = (h->n_units + 31) / 32;
    dim3 grid ((nwarps + PPM_WARPS - 1) / PPM_WARPS), blk (PPM_WARPS * 32);
#define PPM_GO(K, A) ppm_kernel<K, A><<<grid, blk, smem, st>>> (d_in, stride, (int)h->n_units, (int)nfram, h->pr, h->d_mv, h->d_z1, h->d_z2, h->d_m, h->d_res)
    if (h->kind == B200M_PPM_VU) { if (al) PPM_GO (0, true); else PPM_GO (0, false); }
    else if (h->kind == B200M_PPM_MS) { if (al) PPM_GO (3, true); else PPM_GO (3, false); }
    else { if (al) PPM_GO (1, true); else PPM_GO (1, false); }
#undef PPM_GO
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
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags (&h->own, cudaStreamNonBlocking);
    const int smem_max = PPM_WARPS * PPM_STAGES * 2 * PPM_PLANE * (int)sizeof (float);
#define PPM_ATTR(K, A) if (e == cudaSuccess) e = cudaFuncSetAttribute (ppm_kernel<K, A>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max)
    PPM_ATTR (0, true); PPM_ATTR (0, false); PPM_ATTR (1, true); PPM_ATTR (1, false); PPM_ATTR (3, true); PPM_ATTR (3, false);
#undef PPM_ATTR
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
    cudaFree (h->d_z1); cudaFree (h->d_z2); cudaFree (h->d_m); cudaFree (h->d_out); cudaFree (h->d_res); cudaFree (h->d_mv); h->stage.release ();
    if (h->own) cudaStreamDestroy (h->own);
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
    ppm_clear_kernel<<<(nm + 255) / 256, 256, 0, ppm_stream (h, stream)>>> (m0, nm, h->d_z1, h->d_z2, h->d_m, h->d_out, h->d_res);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    if (h->kind == B200M_PPM_MS) {                         // the constructor's gains: a fresh Msppmdsp (-6) pair
        const uint32_t u0 = unit < 0 ? 0 : (uint32_t)unit, u1 = unit < 0 ? h->n_units : u0 + 1;
        for (uint32_t u = u0; u < u1; ++u) { h->db[u] = make_float2 (0, 0); h->mv[u] = make_float2 (1, 1); }
        return b200m_ppm_set_gain_inst (h, unit, -6, -6);
    }
    return 0;
}

int b200m_ppm_process_device (b200m_ppm* h, const float* d_in, size_t stride, uint32_t nfram, void* stream)
{
    if (int rc = check_block_args (h, d_in, stride, nfram)) return rc;
    DeviceGuard g (h->device);
    h->last_host = false;
    return ppm_process (h, d_in, stride, nfram, (cudaStream_t)stream);
}

int b200m_ppm_process_host (b200m_ppm* h, const float* in, size_t stride, uint32_t nfram)
{
    if (int rc = check_block_args (h, in, stride, nfram)) return rc;
    DeviceGuard g (h->device);
    B200M_ENTER_HOST_PATH (h);
    const size_t rows = h->kind == B200M_PPM_MS ? (size_t)2 * h->n_units : h->n_units;
    if (h->stage.ensure (rows, nfram)) return set_err (B200M_E_NOMEM, "staging buffer allocation failed");
    B200M_CUDA (cudaMemcpy2DAsync (h->stage.d, h->stage.cap * sizeof (float), in, stride * sizeof (float),
                                   (size_t)nfram * sizeof (float), rows, cudaMemcpyHostToDevice, h->own));
    h->last_host = true;
    return ppm_process (h, h->stage.d, h->stage.cap, nfram, h->own);
}

int b200m_ppm_read_device (b200m_ppm* h, void* stream)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    DeviceGuard g (h->device);
    ppm_read_kernel<<<(h->n_meters + 255) / 256, 256, 0, ppm_stream (h, stream)>>> ((int)h->n_meters, h->g, h->d_m, h->d_res, h->d_out);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}

int b200m_ppm_results (b200m_ppm* h, float* out, void* stream)
{
    if (!h || !out) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = ppm_stream (h, stream);
    B200M_CUDA (cudaMemcpyAsync (out, h->d_out, h->n_meters * sizeof (float), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}

int b200m_ppm_state (b200m_ppm* h, float* state4, void* stream)
{
    if (!h || !state4) return set_err (B200M_E_INVAL, "NULL argument");
    DeviceGuard g (h->device);
    cudaStream_t st = ppm_stream (h, stream);
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

}  // extern "C"
