// host_common.cu — error reporting, launch accounting and pinned-memory helpers of the C ABI.
#include <ctype.h>
#include <sched.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "common.cuh"

namespace b200m {

thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};

int set_err (int code, const char* fmt, ...)
{
    va_list ap; va_start (ap, fmt);
    vsnprintf (g_err, sizeof (g_err), fmt, ap);
    va_end (ap);
    return code;
}

int cuda_fail (cudaError_t e, const char* what, const char* file, int line)
{
    const char* base = strrchr (file, '/');
    snprintf (g_err, sizeof (g_err), "CUDA error %d (%s) in %s at %s:%d", (int)e, cudaGetErrorString (e), what, base ? base + 1 : file, line);
    cudaGetLastError ();   // clear the sticky-free error state
    return (e == cudaErrorMemoryAllocation) ? B200M_E_NOMEM
         : (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) ? B200M_E_NODEVICE : B200M_E_CUDA;
}

int check_block_args (const void* h, const void* in, size_t stride, uint32_t nfram)
{
    if (!h) return set_err (B200M_E_INVAL, "NULL handle");
    if (!in) return set_err (B200M_E_INVAL, "NULL input");
    if (nfram == 0 || nfram > B200M_MAX_BLOCK) return set_err (B200M_E_INVAL, "nfram %u outside 1..%u", nfram, B200M_MAX_BLOCK);
    if (stride < nfram) return set_err (B200M_E_INVAL, "stride %zu < nfram %u", stride, nfram);
    return 0;
}

int ragged_check (uint32_t n, uint32_t nfram, const uint32_t* len)
{
    if (!len) return 0;
    bool rag = false;
    for (uint32_t i = 0; i < n; ++i) {
        if (len[i] > nfram) return set_err (B200M_E_INVAL, "len[%u] = %u exceeds nfram = %u", i, len[i], nfram);
        rag |= len[i] != nfram;
    }
    return rag ? 1 : 0;
}

int group_check (const uint32_t* group, uint32_t n, uint32_t n_groups, uint32_t max_groups)
{
    if (n_groups == 0 || n_groups > max_groups) return set_err (B200M_E_INVAL, "n_groups %u outside 1..%u", n_groups, max_groups);
    for (uint32_t i = 0; i < n; ++i)
        if (group[i] >= n_groups && group[i] != B200M_NO_GROUP)
            return set_err (B200M_E_INVAL, "group[%u] = %u is neither < n_groups = %u nor B200M_NO_GROUP", i, group[i], n_groups);
    return 0;
}

int GroupList::assign (const uint32_t* group, uint32_t n, uint32_t ng, uint32_t max_groups, cudaStream_t st)
{
    if (!of.empty () && ng == n_groups && !memcmp (group, of.data (), n * sizeof (uint32_t))) return 0;
    cudaError_t e = cudaSuccess;
    uint32_t* w = up.stage (2 * (size_t)n + max_groups + 1, &e);
    if (!w) return cuda_fail (e, "GroupList::assign", __FILE__, __LINE__);
    std::vector<uint32_t> off (ng + 1, 0);
    for (uint32_t i = 0; i < n; ++i) if (group[i] != B200M_NO_GROUP) off[group[i] + 1]++;
    for (uint32_t a = 0; a < ng; ++a) off[a + 1] += off[a];
    const uint32_t nm = off[ng];
    memcpy (w + 2 * (size_t)nm, off.data (), (ng + 1) * sizeof (uint32_t));
    for (uint32_t i = 0; i < n; ++i)
        if (group[i] != B200M_NO_GROUP) { const uint32_t p = off[group[i]]++; w[p] = i; w[nm + p] = group[i]; }
    B200M_CUDA (up.upload (2 * (size_t)nm + ng + 1, st));
    of.assign (group, group + n); n_groups = ng; members = nm;
    return 0;
}

int BankPath::enter_device ()
{
    if (last_host) B200M_CUDA (cudaStreamSynchronize (own));
    last_host = false;
    return 0;
}

int BankPath::enter_host ()
{
    if (!last_host) B200M_CUDA (cudaDeviceSynchronize ());
    last_host = true;
    return 0;
}

int BankPath::stage_block (const float* in, size_t stride, uint32_t nfram, size_t rows, cudaStream_t st, const float** d, size_t* dstride)
{
    if (int rc = enter_host ()) return rc;
    if (stage.ensure (rows, nfram)) return set_err (B200M_E_NOMEM, "staging buffer allocation failed");
    B200M_CUDA (cudaMemcpy2DAsync (stage.d, stage.cap * sizeof (float), in, stride * sizeof (float), (size_t)nfram * sizeof (float), rows,
                                   cudaMemcpyHostToDevice, st));
    *d = stage.d; *dstride = stage.cap;
    return 0;
}

void BankPath::release ()
{
    stage.release ();
    if (own) cudaStreamDestroy (own);
    own = nullptr;
}

}  // namespace b200m

using namespace b200m;

extern "C" {

int b200m_abi_version (void) { return B200M_ABI_VERSION; }
const char* b200m_last_error (void) { return g_err; }

int b200m_device_count (void)
{
    int n = 0;
    if (cudaGetDeviceCount (&n) != cudaSuccess) { cudaGetLastError (); return 0; }
    return n;
}

// Pinned staging memory should sit on the NUMA node the GPU hangs off: a buffer on the other socket halves the H2D rate
// (the copy crosses the inter-socket link).  Pages are placed where the allocating thread runs (first touch), so the
// calling thread is moved onto the GPU-local CPUs for the duration of the allocation.  B200M_NUMA_BIND=0 disables this.
static bool gpu_local_cpus (cpu_set_t* set)
{
    int dev = 0; char bus[32] = {0};
    if (cudaGetDevice (&dev) != cudaSuccess || cudaDeviceGetPCIBusId (bus, sizeof (bus), dev) != cudaSuccess) return false;
    for (char* c = bus; *c; ++c) *c = (char)tolower (*c);
    char path[128]; snprintf (path, sizeof (path), "/sys/bus/pci/devices/%s/local_cpulist", bus);
    FILE* f = fopen (path, "r");
    if (!f) return false;
    char line[1024] = {0};
    const bool got = fgets (line, sizeof (line), f) != nullptr;
    fclose (f);
    if (!got) return false;
    CPU_ZERO (set);
    int n = 0;
    char* save = nullptr;
    for (char* tok = strtok_r (line, ",\n", &save); tok; tok = strtok_r (nullptr, ",\n", &save)) {      // "0-31,64-95"
        int a = 0, b = 0;
        const int k = sscanf (tok, "%d-%d", &a, &b);
        if (k < 1) continue;
        if (k == 1) b = a;
        for (int c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET (c, set); ++n; }
    }
    return n > 0;
}

int b200m_host_alloc (void** p, size_t bytes)
{
    if (!p) return set_err (B200M_E_INVAL, "NULL out pointer");
    cpu_set_t old_set, local;
    bool moved = false;
    const char* v = getenv ("B200M_NUMA_BIND");
    if (!(v && atoi (v) == 0) && sched_getaffinity (0, sizeof (old_set), &old_set) == 0 && gpu_local_cpus (&local)) {
        cpu_set_t both;
        CPU_AND (&both, &old_set, &local);                      // never leave the set the caller was confined to
        if (CPU_COUNT (&both) > 0) moved = sched_setaffinity (0, sizeof (both), &both) == 0;
    }
    const cudaError_t e = cudaHostAlloc (p, bytes, cudaHostAllocDefault);
    if (moved) sched_setaffinity (0, sizeof (old_set), &old_set);
    B200M_CUDA (e);
    return 0;
}

int b200m_host_free (void* p)
{
    if (!p) return 0;
    B200M_CUDA (cudaFreeHost (p));
    return 0;
}

uint64_t b200m_launch_count (void) { return g_launches.load (); }

}
