// common.cuh — shared host/device helpers of the b200meters CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <new>
#include <type_traits>
#include <vector>

#include "../../include/b200meters.h"

namespace b200m {

// Run-time choices handed to a template as compile-time ones, for the host code that picks a kernel instantiation.
// with_bools (f, b...) calls f (std::bool_constant<b> {}...); f is instantiated for every combination.
template <class F> auto with_bools (F f) { return f (); }
template <class F, class... B> auto with_bools (F f, bool b, B... bs)
{
    auto g = [&] (auto c) { return with_bools ([&] (auto... cs) { return f (c, cs...); }, bs...); };
    return b ? g (std::true_type {}) : g (std::false_type {});
}
// with_int<V...> (v, f) calls f (std::integral_constant<int, v> {}) if v is one of V..., else with the last of them
template <int V, int... Vs, class F> auto with_int (int v, F f)
{
    if constexpr (sizeof... (Vs) == 0) return f (std::integral_constant<int, V> {});
    else return v == V ? f (std::integral_constant<int, V> {}) : with_int<Vs...> (v, f);
}

// ---------------------------------------------------------------- host-side plumbing
extern thread_local char g_err[512];
extern std::atomic<uint64_t> g_launches;

int  set_err (int code, const char* fmt, ...);
int  cuda_fail (cudaError_t e, const char* what, const char* file, int line);

#define B200M_CUDA(call)                                                             \
    do {                                                                             \
        cudaError_t e_ = (call);                                                     \
        if (e_ != cudaSuccess) return b200m::cuda_fail (e_, #call, __FILE__, __LINE__); \
    } while (0)

#define B200M_LAUNCHED(n) (b200m::g_launches.fetch_add ((n), std::memory_order_relaxed))

// every bank pins its device on entry and restores the caller's device on exit
struct DeviceGuard {
    int prev = -1; bool ok = true;
    explicit DeviceGuard (int dev) {
        if (cudaGetDevice (&prev) != cudaSuccess) { ok = false; return; }
        if (prev != dev && cudaSetDevice (dev) != cudaSuccess) ok = false;
    }
    ~DeviceGuard () { if (prev >= 0) cudaSetDevice (prev); }
};

// device staging area for *_process_host: [channels][cap] floats, grown on demand
struct HostStage {
    float* d = nullptr; size_t chans = 0, cap = 0;
    int ensure (size_t channels, size_t n) {
        if (d && channels == chans && n <= cap) return 0;
        if (d) { cudaFree (d); d = nullptr; }
        size_t c = (n + 63) & ~size_t (63);
        if (cudaMalloc (&d, channels * c * sizeof (float)) != cudaSuccess) { d = nullptr; return B200M_E_NOMEM; }
        chans = channels; cap = c; return 0;
    }
    void release () { if (d) cudaFree (d); d = nullptr; }
};

int check_block_args (const void* h, const void* in, size_t stride, uint32_t nfram);

// A ragged block (b200m_*_ragged_*): len[i] <= nfram frames for each of n meters or instances.  1 if some len[i] differs from
// nfram, 0 if none does or len is NULL (the plain call), B200M_E_INVAL if one exceeds nfram (nothing is enqueued then).
int ragged_check (uint32_t n, uint32_t nfram, const uint32_t* len);

// Upload of a ragged block's per-row words (lengths, and whatever a bank derives from them): a device array and two pinned host
// slots, allocated with the first ragged block.  The copy from one slot may still be queued while the next block fills the other;
// stage() waits until the slot's previous copy has run, so a pinned copy is truly asynchronous and never sees its source change.
struct RaggedLen {
    uint32_t* d = nullptr; uint32_t* h[2] = {nullptr, nullptr}; cudaEvent_t ev[2] = {nullptr, nullptr}; int slot = 0;
    // the host slot for the next upload (room for `cap` words, the same every call), or nullptr with the CUDA error in *err
    uint32_t* stage (size_t cap, cudaError_t* err) {
        cudaError_t e = cudaSuccess;
        if (!d) e = cudaMalloc ((void**)&d, cap * sizeof (uint32_t));
        for (int s = 0; s < 2; ++s) {
            if (e == cudaSuccess && !h[s]) e = cudaHostAlloc ((void**)&h[s], cap * sizeof (uint32_t), cudaHostAllocDefault);
            if (e == cudaSuccess && !ev[s]) e = cudaEventCreateWithFlags (&ev[s], cudaEventDisableTiming);
        }
        if (e == cudaSuccess) e = cudaEventSynchronize (ev[slot]);
        *err = e;
        return e == cudaSuccess ? h[slot] : nullptr;
    }
    // enqueue the copy of the first `words` words of the slot stage() returned to d, on `st`; the next stage() takes the other slot
    cudaError_t upload (size_t words, cudaStream_t st) {
        cudaError_t e = cudaMemcpyAsync (d, h[slot], words * sizeof (uint32_t), cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaEventRecord (ev[slot], st);
        slot ^= 1;
        return e;
    }
    // stage() + the copy of len[0 .. n) + upload() on `st`: 0 with the lengths in d, or the error (set_err)
    int put (const uint32_t* len, size_t n, cudaStream_t st) {
        cudaError_t e = cudaSuccess;
        if (uint32_t* hl = stage (n, &e)) { memcpy (hl, len, n * sizeof (uint32_t)); e = upload (n, st); }
        return e == cudaSuccess ? 0 : cuda_fail (e, "RaggedLen::put", __FILE__, __LINE__);
    }
    void release () {
        if (d) cudaFree (d);
        for (int s = 0; s < 2; ++s) { if (h[s]) cudaFreeHost (h[s]); if (ev[s]) cudaEventDestroy (ev[s]); h[s] = nullptr; ev[s] = nullptr; }
        d = nullptr;
    }
};

// The album member list of b200m_ebu_group_reduce and b200m_dr14_group_reduce.  group (host, n entries) maps instance i to an
// album 0 .. n_groups - 1 or to B200M_NO_GROUP.  group_check refuses n_groups outside 1 .. max_groups or an album id out of range
// (B200M_E_INVAL; the caller has checked its pointers).  assign sorts the instances by album (a counting sort, each album's
// members in instance order) and uploads in one copy the member list, each member's album, and each album's offset into the list
// (n_groups + 1 words: album a's members are members[off[a] .. off[a + 1])).  It uploads nothing when group and n_groups are the
// previous call's.
int group_check (const uint32_t* group, uint32_t n, uint32_t n_groups, uint32_t max_groups);

struct GroupList {
    std::vector<uint32_t> of;                // the assignment as last uploaded (empty: none yet)
    uint32_t n_groups = 0, members = 0;      // its album count and number of members
    RaggedLen up;                            // up.d: members [members], album [members], off [n_groups + 1]
    const uint32_t* d_members () const { return up.d; }
    const uint32_t* d_album () const { return up.d + members; }
    const uint32_t* d_off () const { return up.d + 2 * (size_t)members; }
    // max_groups: the bank's cap on n_groups, the same every call (it sizes the upload buffers)
    int assign (const uint32_t* group, uint32_t n, uint32_t n_groups, uint32_t max_groups, cudaStream_t st);
    void release () { up.release (); of.clear (); }
};

// The host/device path policy of a bank, the one place that keeps the ordering promise of include/b200meters.h (Conventions).
// A bank switches to its own stream with the first *_host call; whatever the caller queued before that (controls on the streams it
// passed) must not race with it: one device-wide synchronisation at the transition, nothing afterwards.  And back: the bank's own
// stream does not synchronise with the caller's, so the first *_device call after *_host calls waits for the own stream on the host
// (the host path's copies and kernels have then run); one wait at the transition, nothing afterwards.
struct BankPath {
    cudaStream_t own = nullptr;          // the host path's copies and kernels
    HostStage stage;                     // the device copy of a host-path block
    bool last_host = false;              // the bank was last driven on the host path
    // the stream of getters and controls: the bank's own after a host-path call, else the caller's
    cudaStream_t stream (void* caller) const { return last_host ? own : (cudaStream_t)caller; }
    int enter_device ();                 // every device-path call; waits for own at the switch
    int enter_host ();                   // every host-path call; synchronises the device at the switch
    // enter_host, then the copy of a host block (rows x nfram, row pitch stride) into the stage on `st` (normally own):
    // *d / *dstride are the staged block
    int stage_block (const float* in, size_t stride, uint32_t nfram, size_t rows, cudaStream_t st, const float** d, size_t* dstride);
    void release ();                     // frees the stage and destroys own
};

inline int no_check () { return 0; }

// The point log of a bank (the EBU R128 loudness log, the DR-14 window log): one point of NF floats per completed fragment or window
// of an instance, `cap` points per instance in a ring on the device.  Field f of point slot s of instance i is
// pts[(f * cap + s) * n_inst + i] (planes [NF][cap][n_inst]: lane = instance stores coalesce); written[i] counts the instance's
// points, the next goes to slot written[i] % cap.  pts == nullptr: the log is off.
struct PointLog { float* pts; unsigned long long* written; uint32_t cap; };

// The host side of a point log: the planes and counters the bank's kernels update, the read cursors, and the drain's device output
// (points, counts, lost counts).
struct PointRing {
    PointLog log = {nullptr, nullptr, 0};
    unsigned long long *rd = nullptr, *lost = nullptr; float* out = nullptr; uint32_t* cnt = nullptr;
    // an empty log of cap points of nf floats for each of n instances, emptied on st; on an error nothing stays allocated
    cudaError_t alloc (size_t n, uint32_t cap, size_t nf, cudaStream_t st) {
        const size_t pts = (size_t)cap * n * nf * sizeof (float);
        log.cap = cap;
        cudaError_t e = cudaMalloc ((void**)&log.pts, pts);
        if (e == cudaSuccess) e = cudaMalloc ((void**)&log.written, n * sizeof (unsigned long long));
        if (e == cudaSuccess) e = cudaMalloc ((void**)&rd, n * sizeof (unsigned long long));
        if (e == cudaSuccess) e = cudaMalloc ((void**)&lost, n * sizeof (unsigned long long));
        if (e == cudaSuccess) e = cudaMalloc ((void**)&cnt, n * sizeof (uint32_t));
        if (e == cudaSuccess) e = cudaMalloc ((void**)&out, pts);
        if (e == cudaSuccess) e = cudaMemsetAsync (log.written, 0, n * sizeof (unsigned long long), st);
        if (e == cudaSuccess) e = cudaMemsetAsync (rd, 0, n * sizeof (unsigned long long), st);
        if (e != cudaSuccess) release ();
        return e;
    }
    void release () {
        cudaFree (log.pts); cudaFree (log.written); cudaFree (rd); cudaFree (lost); cudaFree (out); cudaFree (cnt);
        log = {nullptr, nullptr, 0}; rd = lost = nullptr; out = nullptr; cnt = nullptr;
    }
};

// One block call of a bank: the body of every *_process_* / *_run_* entry point, plain, _ctl_ and ragged, on both paths.  In order:
// the block arguments; the bank's own check () (0 or an error); the n_len lengths `len` (NULL: every row runs nfram); the device,
// the path switch and, on the host path, the staging copy of `rows` rows onto own (rows == 0: the bank copies the block itself).
// Then run (d_in, stride, st, rlen): rlen is len if some length differs from nfram, else nullptr, and the call takes the plain
// code path.  A refused call enqueues nothing and leaves the bank on its path.  rows and n_len are read from the handle by the
// caller, which passes 0 for a NULL handle: the handle is dereferenced only after check_block_args.
template <class Bank, class Check, class Run>
int bank_call (Bank* h, const float* in, size_t stride, uint32_t nfram, bool host, void* stream, size_t rows, uint32_t n_len,
               const uint32_t* len, Check check, Run run)
{
    if (int rc = check_block_args (h, in, stride, nfram)) return rc;
    if (int rc = check ()) return rc;
    const int rag = ragged_check (n_len, nfram, len);
    if (rag < 0) return rag;
    DeviceGuard g (h->device);
    BankPath& p = h->path;
    const float* d = in; size_t ds = stride; cudaStream_t st = (cudaStream_t)stream;
    if (!host) { if (int rc = p.enter_device ()) return rc; }
    else {
        st = p.own;
        if (int rc = rows ? p.stage_block (in, stride, nfram, rows, st, &d, &ds) : p.enter_host ()) return rc;
    }
    return run (d, ds, st, rag ? len : nullptr);
}

#ifdef __CUDACC__
// ---------------------------------------------------------------- device helpers
#define B200M_DEV __device__ __forceinline__

B200M_DEV bool finitef_ (float v) { return fabsf (v) <= 3.402823466e+38f; }   // false for NaN, +-Inf
B200M_DEV float scrub (float v) { return finitef_ (v) ? v : 0.0f; }           // "!isfinite(z) ? 0 : z"

// cp.async (LDGSTS): global -> shared without a register round trip
B200M_DEV void cp_async16 (void* smem, const void* gmem, int src_bytes) {
    unsigned s = (unsigned)__cvta_generic_to_shared (smem);
    asm volatile ("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(src_bytes));
}
B200M_DEV void cp_async4 (void* smem, const void* gmem, int src_bytes) {
    unsigned s = (unsigned)__cvta_generic_to_shared (smem);
    asm volatile ("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(s), "l"(gmem), "r"(src_bytes));
}
B200M_DEV void cp_async_commit () { asm volatile ("cp.async.commit_group;\n" ::); }
template <int N> B200M_DEV void cp_async_wait () { asm volatile ("cp.async.wait_group %0;\n" ::"n"(N)); }

// ---- log10f, bit-identical to glibc 2.39 libm ------------------------------------------
// The reference turns fragment powers into loudness with log10f (ebumeter/ebu_r128_proc.cc:259,
// :116-122,:140-141) and bins the result into INTEGER histograms (:66-79), so the engine needs
// the host libm's log10f to the last bit, not CUDA's 2-ulp one.  glibc 2.39's log10f is the
// fdlibm wrapper  z = y*log10_2lo + ivln10*logf(x'); return z + y*log10_2hi  (float arithmetic)
// around the table-driven double-precision logf of ARM's optimized-routines (16-entry table,
// degree-3 polynomial).  Both are restated here from the published algorithms; the table is the
// one in libm's __logf_data.  Checked exhaustively on the host (all 2^31 non-negative floats)
// against libm's logf and log10f in FMA and non-FMA form: 0 mismatches — see DESIGN.md §log10f
// and tests/test_libm_parity.py.
static __device__ __constant__ double c_logf_tab[16][2] = {
    {0x1.661ec79f8f3bep+0, -0x1.57bf7808caadep-2}, {0x1.571ed4aaf883dp+0, -0x1.2bef0a7c06ddbp-2},
    {0x1.49539f0f010bp+0, -0x1.01eae7f513a67p-2},  {0x1.3c995b0b80385p+0, -0x1.b31d8a68224e9p-3},
    {0x1.30d190c8864a5p+0, -0x1.6574f0ac07758p-3}, {0x1.25e227b0b8eap+0, -0x1.1aa2bc79c81p-3},
    {0x1.1bb4a4a1a343fp+0, -0x1.a4e76ce8c0e5ep-4}, {0x1.12358f08ae5bap+0, -0x1.1973c5a611cccp-4},
    {0x1.0953f419900a7p+0, -0x1.252f438e10c1ep-5}, {0x1p+0, 0x0p+0},
    {0x1.e608cfd9a47acp-1, 0x1.aa5aa5df25984p-5},  {0x1.ca4b31f026aap-1, 0x1.c5e53aa362eb4p-4},
    {0x1.b2036576afce6p-1, 0x1.526e57720db08p-3},  {0x1.9c2d163a1aa2dp-1, 0x1.bc2860d22477p-3},
    {0x1.886e6037841edp-1, 0x1.1058bc8a07ee1p-2},  {0x1.767dcf5534862p-1, 0x1.4043057b6ee09p-2}};

// logf for x with a normal, positive, finite bit pattern (the wrapper below guarantees it)
B200M_DEV float logf_glibc_normal (float x)
{
    uint32_t ix = __float_as_uint (x);
    if (ix == 0x3f800000u) return 0.0f;
    uint32_t tmp = ix - 0x3f330000u;
    int i = (tmp >> 19) & 15;
    int k = (int32_t)tmp >> 23;
    uint32_t iz = ix - (tmp & 0xff800000u);
    double invc = c_logf_tab[i][0], logc = c_logf_tab[i][1];
    double z = (double)__uint_as_float (iz);
    double r  = __fma_rn (z, invc, -1.0);
    double y0 = __fma_rn ((double)k, 0x1.62e42fefa39efp-1, logc);
    double r2 = __dmul_rn (r, r);
    double y  = __fma_rn (0x1.5575b0be00b6ap-2, r, -0x1.ffffef20a4123p-2);
    y = __fma_rn (-0x1.00ea348b88334p-2, r2, y);
    y = __fma_rn (y, r2, __dadd_rn (y0, r));
    return __double2float_rn (y);
}

B200M_DEV float log10f_glibc (float x)
{
    const float two25 = 3.3554432000e+07f, ivln10 = 4.3429449201e-01f;
    const float log10_2hi = 3.0102920532e-01f, log10_2lo = 7.9034151668e-07f;
    int32_t hx = __float_as_int (x), k = 0;
    if (hx < 0x00800000) {                                  // x < 2^-126, zero or negative
        if ((hx & 0x7fffffff) == 0) return __fdiv_rn (-two25, fabsf (x));      // -inf
        if (hx < 0) return __fdiv_rn (__fsub_rn (x, x), __fsub_rn (x, x));     // NaN
        k -= 25; x = __fmul_rn (x, two25); hx = __float_as_int (x);
    }
    if (hx >= 0x7f800000) return __fadd_rn (x, x);
    k += (hx >> 23) - 127;
    int32_t i = (int32_t)(((uint32_t)k & 0x80000000u) >> 31);
    hx = (hx & 0x007fffff) | ((0x7f - i) << 23);
    float y = (float)(k + i);
    float z = __fadd_rn (__fmul_rn (y, log10_2lo), __fmul_rn (ivln10, logf_glibc_normal (__int_as_float (hx))));
    return __fadd_rn (z, __fmul_rn (y, log10_2hi));
}

// ---- drain of a point log (PointLog) ---------------------------------------------------
// Per instance the points written since the last drain, oldest first, at most cap of them, into out[n_inst][cap][NF] (NaN past the
// instance's count), with count[i] and lost[i] (unread points overwritten before this drain); then the read cursor moves to
// written[i].  A CTA owns 32 instances and walks their points in tiles of PTS: lane = instance reads the planes, a shared-memory
// transpose makes the stores of the [cap][NF] rows coalesce.  The static tile is 32 x (PTS * NF + 1) floats, under 48 KB: PTS = 32
// up to NF = 11, PTS = 16 up to NF = 23.
constexpr int LOG_DRAIN_ROWS = 8;

template <int NF, int PTS>
__global__ void __launch_bounds__ (32 * LOG_DRAIN_ROWS)
log_drain_kernel (int n_inst, PointLog lg, unsigned long long* __restrict__ rd, float* __restrict__ out, uint32_t* __restrict__ count,
                  unsigned long long* __restrict__ lost)
{
    __shared__ float tile[32][PTS * NF + 1];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int i0 = blockIdx.x * 32, i = i0 + tx;
    const uint32_t cap = lg.cap;
    const size_t pl = (size_t)cap * n_inst;
    unsigned long long w = 0, start = 0;
    uint32_t cnt = 0;
    if (i < n_inst) {
        w = lg.written[i];
        const unsigned long long unread = w - rd[i];
        cnt = unread < cap ? (uint32_t)unread : cap;
        start = w - cnt;
        if (ty == 0) { count[i] = cnt; lost[i] = unread - cnt; }
    }
    for (uint32_t j0 = 0; j0 < cap; j0 += PTS) {
        for (int jl = ty; jl < PTS; jl += LOG_DRAIN_ROWS) {
            const uint32_t j = j0 + jl;
            float v[NF];
            if (i < n_inst && j < cnt) {
                const float* p = lg.pts + (size_t)((start + j) % cap) * n_inst + i;
#pragma unroll
                for (int f = 0; f < NF; ++f) v[f] = p[f * pl];
            } else {
#pragma unroll
                for (int f = 0; f < NF; ++f) v[f] = __int_as_float (0x7fc00000);
            }
#pragma unroll
            for (int f = 0; f < NF; ++f) tile[tx][jl * NF + f] = v[f];
        }
        __syncthreads ();
        const int nq = (int)min ((uint32_t)PTS, cap - j0) * NF;      // the tile's floats of one instance's row, contiguous in out
        for (int il = ty; il < 32 && i0 + il < n_inst; il += LOG_DRAIN_ROWS) {
            float* o = out + ((size_t)(i0 + il) * cap + j0) * NF;
            for (int q = tx; q < nq; q += 32) o[q] = tile[il][q];
        }
        __syncthreads ();
    }
    if (i < n_inst && ty == 0) rd[i] = w;
}

// b200m_*_log_drain of n instances on st: the drain kernel, the copies of its output into the host arrays out [n][cap][NF],
// count [n] and lost [n], and the wait for them
template <int NF, int PTS>
int log_drain (PointRing& r, size_t n, float* out, uint32_t* count, uint64_t* lost, cudaStream_t st)
{
    log_drain_kernel<NF, PTS><<<(unsigned)((n + 31) / 32), 32 * LOG_DRAIN_ROWS, 0, st>>> ((int)n, r.log, r.rd, r.out, r.cnt, r.lost);
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    B200M_CUDA (cudaMemcpyAsync (out, r.out, n * r.log.cap * NF * sizeof (float), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaMemcpyAsync (count, r.cnt, n * sizeof (uint32_t), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaMemcpyAsync (lost, r.lost, n * sizeof (uint64_t), cudaMemcpyDeviceToHost, st));
    B200M_CUDA (cudaStreamSynchronize (st));
    return 0;
}
#endif  // __CUDACC__

}  // namespace b200m
