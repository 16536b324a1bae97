// pcm.cu — interleaved integer / float PCM to the planar float32 rows every bank reads (b200m_pcm_planar_device).
//
// A decoded file is interleaved PCM, frames [t][c] of 2, 3 or 4 bytes per sample.  One launch converts a block of N clips: clip i
// starts at in + i * in_stride and holds nfram frames of nchan samples; output row k = i * nchan + c, frame t, is
// scale (sample (t, c) of clip i), scale = 2^-(bits - 1) (F32: a bit copy).  Every conversion is exact: an int16 or a sign-extended
// 24-bit value is exact in float, and the power-of-two scale is one exact multiply (S32 rounds x to nearest-even first).
//
// The kernel is memory bound: it reads bps bytes and writes 4 bytes per sample.  A CTA owns one tile of TF frames of one clip:
//  - it stages the tile's contiguous bytes in shared memory with 16-byte loads, and single-byte loads for the at most 15 bytes
//    before the first and after the last 16-byte boundary of the tile (`in` need only be a multiple of the sample size, 1 byte
//    for S24, so a whole WAV data chunk can be converted where it lies).  Shared memory mirrors the global 16-byte grid: byte g of
//    the tile sits at (g + head) with head = the tile's start address mod 16, so each 16-byte load lands on a 16-byte slot;
//  - then each warp writes 32 consecutive frames of one row, one coalesced 128-byte line.  A warp reads one channel of 32 frames,
//    a shared-memory stride of nchan * bps bytes; the 16-byte slots of each 128-byte line are XOR-swizzled by the line index so
//    that strides of 64 or 128 bytes (16 or 32 channels) spread over 8 slots instead of one bank.
#include <algorithm>
#include "common.cuh"

namespace b200m {

constexpr int PCM_THREADS = 256;
constexpr size_t PCM_TILE_BYTES = 16384;           // staged bytes per CTA at most: 8 CTAs of 256 threads fit one SM

__host__ __device__ constexpr uint32_t pcm_bps (int fmt) { return fmt == B200M_PCM_S16 ? 2u : fmt == B200M_PCM_S24 ? 3u : 4u; }

// the shared-memory byte of staged byte b: 16-byte slot (b >> 4) & 7 of 128-byte line b >> 7 XORed with the line's low 3 bits
__device__ __forceinline__ uint32_t pcm_sw (uint32_t b) { return b ^ (((b >> 7) & 7u) << 4); }

template <int FMT>
__device__ __forceinline__ float pcm_sample (const uint8_t* s, uint32_t b)
{
    if constexpr (FMT == B200M_PCM_S16) {
        return (float)*(const int16_t*)(s + pcm_sw (b)) * 0x1p-15f;
    } else if constexpr (FMT == B200M_PCM_S24) {
        const uint32_t u = (uint32_t)s[pcm_sw (b)] | (uint32_t)s[pcm_sw (b + 1)] << 8 | (uint32_t)s[pcm_sw (b + 2)] << 16;
        return (float)((int32_t)(u << 8) >> 8) * 0x1p-23f;
    } else if constexpr (FMT == B200M_PCM_S32) {
        return __int2float_rn (*(const int32_t*)(s + pcm_sw (b))) * 0x1p-31f;
    } else {
        return __uint_as_float (*(const uint32_t*)(s + pcm_sw (b)));
    }
}

// tiles: tiles per clip, each of tf frames (a multiple of 32), the last one short
template <int FMT>
__global__ void __launch_bounds__ (PCM_THREADS)
pcm_planar_kernel (const uint8_t* __restrict__ in, size_t in_stride, uint32_t nchan, uint32_t nfram, uint32_t tf, uint32_t tiles,
                   size_t n_tiles, float* __restrict__ out, size_t out_stride)
{
    extern __shared__ __align__ (128) uint8_t sm[];
    constexpr uint32_t bps = pcm_bps (FMT);
    const uint32_t fb = nchan * bps;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (size_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const size_t i = tile / tiles;
        const uint32_t f0 = (uint32_t)(tile - i * tiles) * tf;
        const uint32_t nf = min (tf, nfram - f0);
        const uint8_t* g = in + i * in_stride + (size_t)f0 * fb;
        const uint32_t bytes = nf * fb;
        const uint32_t head = (uint32_t)((uintptr_t)g & 15u);
        // bytes [v0, v1) of the tile are whole 16-byte words in global memory; the rest go one byte at a time
        const uint32_t v0 = min ((16u - head) & 15u, bytes);
        const uint32_t v1 = v0 + ((bytes - v0) & ~15u);
        for (uint32_t b = v0 + threadIdx.x * 16; b < v1; b += PCM_THREADS * 16)
            *(uint4*)(sm + pcm_sw (head + b)) = __ldg ((const uint4*)(g + b));
        if (threadIdx.x < v0) sm[pcm_sw (head + threadIdx.x)] = g[threadIdx.x];
        if (threadIdx.x < bytes - v1) sm[pcm_sw (head + v1 + threadIdx.x)] = g[v1 + threadIdx.x];
        __syncthreads ();
        const uint32_t groups = (nf + 31) >> 5;
        for (uint32_t w = warp; w < nchan * groups; w += PCM_THREADS / 32) {
            const uint32_t c = w / groups, t = ((w - c * groups) << 5) + lane;
            if (t < nf)
                out[((size_t)i * nchan + c) * out_stride + f0 + t] = pcm_sample<FMT> (sm, head + t * fb + c * bps);
        }
        __syncthreads ();
    }
}

}  // namespace b200m

using namespace b200m;

extern "C" int b200m_pcm_planar_device (int device, const void* in, int format, uint32_t n_clips, uint32_t nchan, uint32_t nfram,
                                        size_t in_stride, float* out, size_t out_stride, void* stream)
{
    if (!in || !out) return set_err (B200M_E_INVAL, "NULL pointer");
    if (format < B200M_PCM_S16 || format > B200M_PCM_F32) return set_err (B200M_E_INVAL, "unknown PCM format %d", format);
    if (n_clips == 0) return set_err (B200M_E_INVAL, "n_clips is 0");
    if (nchan == 0 || nchan > B200M_PCM_MAX_CHANNELS) return set_err (B200M_E_INVAL, "nchan %u outside 1..%u", nchan, B200M_PCM_MAX_CHANNELS);
    if (nfram == 0 || nfram > B200M_MAX_BLOCK) return set_err (B200M_E_INVAL, "nfram %u outside 1..%u", nfram, B200M_MAX_BLOCK);
    const uint32_t bps = pcm_bps (format);
    const size_t fb = (size_t)nchan * bps;
    if (in_stride < nfram * fb) return set_err (B200M_E_INVAL, "in_stride %zu < nfram * nchan * %u = %zu bytes", in_stride, bps, nfram * fb);
    const uint32_t align = format == B200M_PCM_S24 ? 1u : bps;       // packed 24-bit samples may start at any byte
    if ((uintptr_t)in % align || in_stride % align) return set_err (B200M_E_INVAL, "in and in_stride must be multiples of %u bytes", align);
    if (out_stride < nfram) return set_err (B200M_E_INVAL, "out_stride %zu < nfram %u", out_stride, nfram);
    if (b200m_device_count () <= 0) return set_err (B200M_E_NODEVICE, "no CUDA device");
    DeviceGuard dg (device);
    if (!dg.ok) return set_err (B200M_E_NODEVICE, "cannot select CUDA device %d", device);
    // tile frames: a multiple of 32 with tf * fb <= PCM_TILE_BYTES (32 channels of 4 bytes: 128 frames), no more than the block needs
    const uint32_t tf = (uint32_t)std::min<size_t> (std::max<size_t> (PCM_TILE_BYTES / fb, 32) & ~size_t (31), (nfram + 31) & ~31u);
    const uint32_t tiles = (nfram + tf - 1) / tf;
    const size_t n_tiles = (size_t)n_clips * tiles;
    const size_t smem = (16 + tf * fb + 127) & ~size_t (127);       // head <= 15 bytes, whole 128-byte swizzle lines
    const unsigned grid = (unsigned)std::min<size_t> (n_tiles, 0x7fffffff);
    const cudaStream_t st = (cudaStream_t)stream;
    const uint8_t* src = (const uint8_t*)in;
    switch (format) {
    case B200M_PCM_S16: pcm_planar_kernel<B200M_PCM_S16><<<grid, PCM_THREADS, smem, st>>> (src, in_stride, nchan, nfram, tf, tiles, n_tiles, out, out_stride); break;
    case B200M_PCM_S24: pcm_planar_kernel<B200M_PCM_S24><<<grid, PCM_THREADS, smem, st>>> (src, in_stride, nchan, nfram, tf, tiles, n_tiles, out, out_stride); break;
    case B200M_PCM_S32: pcm_planar_kernel<B200M_PCM_S32><<<grid, PCM_THREADS, smem, st>>> (src, in_stride, nchan, nfram, tf, tiles, n_tiles, out, out_stride); break;
    default:            pcm_planar_kernel<B200M_PCM_F32><<<grid, PCM_THREADS, smem, st>>> (src, in_stride, nchan, nfram, tf, tiles, n_tiles, out, out_stride); break;
    }
    B200M_LAUNCHED (1);
    B200M_CUDA (cudaGetLastError ());
    return 0;
}
