// f3, read side: the archive reader's gather (sm_90a).
//
// A read of an archive (capi_read.cu) resolves its byte ranges to pieces: the intersections of one range with one
// chunk held in the reader's cache.  A restore of many small files yields hundreds of thousands of pieces per call, and
// one cudaMemcpyAsync per piece would cost microseconds of host time each; K14 copies the whole list in one launch.
//
//   K14 k_read_gather : one warp per tile of READ_TILE bytes of a piece (tile_first: prefix of the pieces' tile counts,
//                       owner_of finds a tile's piece), eight tiles per CTA and a grid-stride loop, so a list of 4 KiB
//                       pieces runs eight pieces per CTA.  Where source and target share their alignment mod 16 the warp
//                       copies 16-byte vectors with a byte head and tail; otherwise 4-byte words, each target word a
//                       funnel shift of two aligned source words.
#include <algorithm>

#include "device.cuh"
#include "internal.cuh"

namespace pbsgpu {

// the warp's copy of `size` bytes from s to d
__device__ __forceinline__ void read_copy_tile(const uint8_t *s, uint8_t *d, uint32_t size, uint32_t lane) {
    if ((((uintptr_t)s ^ (uintptr_t)d) & 15) == 0) {
        uint32_t head = (uint32_t)((16 - ((uintptr_t)d & 15)) & 15);
        if (head > size) head = size;
        if (lane < head) d[lane] = s[lane];
        const uint32_t nv = (size - head) >> 4, tail0 = head + (nv << 4);
        if (lane < size - tail0) d[tail0 + lane] = s[tail0 + lane];
        const uint4 *sv = (const uint4 *)(s + head);
        uint4 *dv = (uint4 *)(d + head);
        uint32_t v = lane;
        for (; v + 96 < nv; v += 128) {   // four loads in flight per lane
            const uint4 a = __ldg(sv + v), b = __ldg(sv + v + 32), c = __ldg(sv + v + 64), e = __ldg(sv + v + 96);
            dv[v] = a; dv[v + 32] = b; dv[v + 64] = c; dv[v + 96] = e;
        }
        for (; v < nv; v += 32) dv[v] = __ldg(sv + v);
        return;
    }
    uint32_t head = (uint32_t)((4 - ((uintptr_t)d & 3)) & 3);
    if (head > size) head = size;
    if (lane < head) d[lane] = s[lane];
    const uint32_t nw = (size - head) >> 2, tail0 = head + (nw << 2);
    if (lane < size - tail0) d[tail0 + lane] = s[tail0 + lane];
    const uint8_t *sp = s + head;
    const uint32_t mis = (uint32_t)((uintptr_t)sp & 3), sh = mis * 8;
    const uint32_t *s32 = (const uint32_t *)(sp - mis);
    uint32_t *d32 = (uint32_t *)(d + head);
    for (uint32_t w = lane; w < nw; w += 32) {
        const uint32_t a0 = __ldg(s32 + w), a1 = mis ? __ldg(s32 + w + 1) : 0u;   // a1 holds bytes this word needs when mis != 0
        d32[w] = __funnelshift_r(a0, a1, sh);
    }
}

__global__ void __launch_bounds__(256) k_read_gather(const ReadPiece *pieces, const uint64_t *tile_first, uint32_t n,
                                                     uint64_t total) {
    const uint32_t lane = threadIdx.x & 31;
    for (uint64_t t = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5); t < total; t += (uint64_t)gridDim.x * 8) {
        const uint32_t p = owner_of(tile_first, n, t);
        const ReadPiece pc = pieces[p];
        const uint64_t at = (t - tile_first[p]) * READ_TILE, rem = pc.len - at;
        read_copy_tile((const uint8_t *)pc.src + at, (uint8_t *)pc.dst + at, rem < READ_TILE ? (uint32_t)rem : READ_TILE, lane);
    }
}

cudaError_t launch_read_gather(const ReadPiece *pieces, const uint64_t *tile_first, uint32_t n, uint64_t total_tiles,
                               int sm_count, cudaStream_t st) {
    if (total_tiles == 0) return cudaSuccess;
    const uint64_t ctas = std::min<uint64_t>((total_tiles + 7) / 8, (uint64_t)sm_count * 8);
    k_read_gather<<<(unsigned)ctas, 256, 0, st>>>(pieces, tile_first, n, total_tiles);
    return cudaGetLastError();
}

}  // namespace pbsgpu
