// compact.cu -- the HBM-bound compaction kernels: execute the tile list the plan kernel wrote.
// Every output byte of every stripped ELF is produced exactly once: copied from the input arena
// (kept section contents), copied from the per-file scratch slot (regenerated Ehdr/Phdr/Shdr
// tables, .shstrtab, merged notes) or zero-filled (the file holes BFD leaves between sections).
//
// Pure byte movement -- no tensor cores.  Roofline: HBM read+write (SURVEY.md 8d).
//   * lb2_compact_tma_kernel  (compact_tma.cu, default) bulk-copy engine path.
//   * lb2_compact_kernel      (this file; LB2_COMPACT_TMA=0, and lb2_corpus_scatter) warp-per-tile, 16-byte
//                             vectorised LDG/STG, 8 loads in flight per lane, byte-granular heads/tails,
//                             funnel-shifted path for tiles whose source and destination are not congruent
//                             mod 16.
//
// Replaces the data movement GNU strip does with read()/write() per file
// (/root/reference/lambdipy/project_build.py:260).
#include "lb2_common.cuh"
#include "copy_device.cuh"

namespace lb2 {

// Persistent grid; every warp strides over the tile list.  Tiles are <= 16 KB and never cross a
// 16 KB boundary of the destination file, so large extents stream as full 128-byte lines.
__global__ void __launch_bounds__(256) lb2_compact_kernel(CompactArgs a) {
  if (a.ctr->overflow) return;
  const unsigned long long n_tiles = a.ctr->n_tiles;
  const int lane = threadIdx.x & 31;
  const unsigned long long warps = (unsigned long long)gridDim.x * (blockDim.x >> 5);
  unsigned long long t = (unsigned long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  // interleave so that consecutive tiles (consecutive memory) go to different SMs at the same time
  for (; t < n_tiles; t += warps) {
    const TileView v = load_tile(a, t);
    if (v.src) warp_copy_tile(v.src, v.dst, v.len, lane);
    else warp_zero_tile(v.dst, v.len, lane);
  }
}

void launch_compact(const CompactArgs &a, int grid, cudaStream_t s) {
  lb2_compact_kernel<<<grid, 256, 0, s>>>(a);
}

}  // namespace lb2
