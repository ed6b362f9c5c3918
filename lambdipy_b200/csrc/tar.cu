// tar.cu -- the member walk of a tar stream in device memory behind lb2_tar_index (api.cu); the walk itself is
// tar_walk.cuh.
//
// One warp walks the archive.  A header block is one 16-byte load per lane into shared memory, its two checksums a
// warp reduction, the all-zero test a vote; every lane then runs the same walk on the same values, so the control flow
// stays uniform.  The chain is sequential by nature: the next header's offset comes from this one's size, so the walk
// costs one dependent HBM load per member.  Gathered ranges that touch are merged, and their bytes are appended to one
// buffer in range order; past either capacity the walk keeps counting and stops writing.
#include "lb2_common.cuh"
#include "tar_walk.cuh"

namespace lb2 {
namespace {
using tarw::Range;

struct WarpIo {
  const uint8_t *tar;
  uint8_t *h;  // the loaded block, in shared memory
  int64_t su = 0, ss = 0;
  bool zero = false;
  Range *ranges;
  uint8_t *bytes;
  uint64_t max_ranges, bytes_cap;
  uint64_t n_ranges = 0, n_bytes = 0, start = 0, end = 0;  // the last range: [start, end)
  int lane;

  __device__ void load(uint64_t off) {
    const uint4 v = __ldg(reinterpret_cast<const uint4 *>(tar + off) + lane);
    reinterpret_cast<uint4 *>(h)[lane] = v;
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    int32_t u = 0, s = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) {
      const uint32_t at = 16 * lane + i;
      const uint32_t b = (w[i >> 2] >> (8 * (i & 3))) & 0xFF;
      if (at < 148 || at >= 156) {
        u += (int32_t)b;
        s += (int32_t)(int8_t)b;
      }
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) {
      u += __shfl_xor_sync(0xFFFFFFFFu, u, d);
      s += __shfl_xor_sync(0xFFFFFFFFu, s, d);
    }
    su = 256 + u;
    ss = 256 + s;
    zero = __all_sync(0xFFFFFFFFu, (v.x | v.y | v.z | v.w) == 0);
    __syncwarp();
  }

  __device__ void gather(uint64_t off, uint64_t len) {
    uint64_t from = off;
    const uint64_t to = off + len;
    if (n_ranges && off <= end) {  // touches the last range: extend it
      if (to <= end) return;
      from = end;
      end = to;
      if (lane == 0 && n_ranges <= max_ranges) ranges[n_ranges - 1].len = end - start;
    } else {
      start = off;
      end = to;
      if (lane == 0 && n_ranges < max_ranges) ranges[n_ranges] = Range{start, len};
      n_ranges++;
    }
    if (n_bytes + (to - from) <= bytes_cap)
      for (uint64_t i = lane; i < to - from; i += 32) bytes[n_bytes + i] = tar[from + i];
    n_bytes += to - from;
  }
};

__global__ void __launch_bounds__(32) lb2_tar_walk_kernel(const uint8_t *tar, uint64_t n, Range *ranges, uint64_t max_ranges,
                                                         uint8_t *bytes, uint64_t bytes_cap, TarWalkOut *out) {
  __shared__ __align__(16) uint8_t block[tarw::BLOCK];
  WarpIo io;
  io.tar = tar;
  io.h = block;
  io.ranges = ranges;
  io.bytes = bytes;
  io.max_ranges = max_ranges;
  io.bytes_cap = bytes_cap;
  io.lane = threadIdx.x & 31;
  tarw::WalkResult r;
  tarw::walk(io, tar, n, r);
  if (io.lane == 0) *out = TarWalkOut{io.n_ranges, io.n_bytes, r.members, r.stop_off, r.reason, 0};
}

}  // namespace

void launch_tar_walk(const uint8_t *tar, uint64_t n, void *ranges, uint64_t max_ranges, uint8_t *bytes, uint64_t bytes_cap,
                     TarWalkOut *out, cudaStream_t s) {
  lb2_tar_walk_kernel<<<1, 32, 0, s>>>(tar, n, static_cast<Range *>(ranges), max_ranges, bytes, bytes_cap, out);
}

}  // namespace lb2
