// f3, read side: the zero-block map of the sparse image restore (sm_90a).
//
// pbsgpu_reader_read_sparse (capi_read.cu) stages the data-chunk bytes of its ranges on the device and asks which
// 4 KiB block parts of them are all zero: those become holes of the restored image, the rest its data extents.  Block b
// of the image is [4096 b, 4096 (b + 1)); a block part is its intersection with one range.  Zero chunks are never
// staged: their block parts are holes by construction, and their bits keep the preset 1.
//
//   K17 k_zero_map : one warp per block part of a staged run (part_first: prefix of the runs' block-part counts,
//                    owner_of finds a part's run), eight parts per CTA and a grid-stride loop.  The warp reads its part
//                    with 16-byte vector loads (a byte head and tail where the part is not 16-byte aligned), two per
//                    lane and step, and votes after each step: a data block usually shows a non-zero byte in its first
//                    1 KiB, so only all-zero parts are read in full.  A part with a non-zero byte clears its bit.
#include <algorithm>

#include "device.cuh"
#include "internal.cuh"

namespace pbsgpu {

// does any of the `size` bytes at s differ from zero?  (warp-uniform result)
__device__ __forceinline__ bool zero_part_nonzero(const uint8_t *s, uint32_t size, uint32_t lane) {
    uint32_t head = (uint32_t)((16 - ((uintptr_t)s & 15)) & 15);
    if (head > size) head = size;
    uint32_t acc = lane < head ? s[lane] : 0u;
    const uint32_t nv = (size - head) >> 4, tail0 = head + (nv << 4);
    if (lane < size - tail0) acc |= s[tail0 + lane];
    const uint4 *sv = (const uint4 *)(s + head);
    for (uint32_t v0 = 0;; v0 += 64) {   // v0: the warp's first vector of this step
        if (__any_sync(0xffffffffu, acc != 0)) return true;
        if (v0 >= nv) return false;
        const uint32_t v = v0 + lane;
        const uint4 a = v < nv ? __ldg(sv + v) : make_uint4(0, 0, 0, 0);
        const uint4 b = v + 32 < nv ? __ldg(sv + v + 32) : make_uint4(0, 0, 0, 0);
        acc = a.x | a.y | a.z | a.w | b.x | b.y | b.z | b.w;
    }
}

__global__ void __launch_bounds__(256) k_zero_map(const ZeroRun *runs, const uint64_t *part_first, uint32_t n,
                                                  uint64_t total, uint32_t *bits) {
    const uint32_t lane = threadIdx.x & 31;
    for (uint64_t t = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5); t < total; t += (uint64_t)gridDim.x * 8) {
        const uint32_t p = owner_of(part_first, n, t);
        const ZeroRun ru = runs[p];
        const uint64_t k = t - part_first[p], blk = ru.off / ZERO_BLOCK + k;
        const uint64_t lo = std::max(ru.off, blk * ZERO_BLOCK), hi = std::min(ru.off + ru.len, (blk + 1) * ZERO_BLOCK);
        if (zero_part_nonzero((const uint8_t *)ru.src + (lo - ru.off), (uint32_t)(hi - lo), lane) && lane == 0) {
            const uint64_t bit = ru.bit + k;
            atomicAnd(bits + (bit >> 5), ~(1u << (bit & 31)));
        }
    }
}

cudaError_t launch_zero_map(const ZeroRun *runs, const uint64_t *part_first, uint32_t n, uint64_t total_parts,
                            uint32_t *bits, int sm_count, cudaStream_t st) {
    if (total_parts == 0) return cudaSuccess;
    const uint64_t ctas = std::min<uint64_t>((total_parts + 7) / 8, (uint64_t)sm_count * 8);
    k_zero_map<<<(unsigned)ctas, 256, 0, st>>>(runs, part_first, n, total_parts, bits);
    return cudaGetLastError();
}

}  // namespace pbsgpu
