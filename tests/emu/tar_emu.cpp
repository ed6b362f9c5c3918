// tar_emu.cpp -- TEST HARNESS: runs the PRODUCT's tar walk (lambdipy_b200/csrc/tar_walk.cuh) on the CPU, one thread
// standing in for the warp of lb2_tar_walk_kernel: the same block loads, checksums and range merging.  It is NOT a CPU
// fallback: it lives under tests/, is built only by the tests and is never loaded by lambdipy_b200/.
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../lambdipy_b200/csrc/tar_walk.cuh"

using namespace lb2::tarw;

struct HostIo {
  const uint8_t *tar;
  uint8_t block[BLOCK];
  const uint8_t *h = block;
  int64_t su = 0, ss = 0;
  bool zero = false;
  std::vector<Range> ranges;
  std::vector<uint8_t> bytes;

  void load(uint64_t off) {
    memcpy(block, tar + off, BLOCK);
    int64_t u = 0, s = 0;
    zero = true;
    for (uint32_t i = 0; i < BLOCK; i++) {
      zero = zero && block[i] == 0;
      if (i < 148 || i >= 156) {
        u += block[i];
        s += (int8_t)block[i];
      }
    }
    su = 256 + u;
    ss = 256 + s;
  }

  void gather(uint64_t off, uint64_t len) {
    uint64_t from = off;
    const uint64_t to = off + len;
    if (!ranges.empty() && off <= ranges.back().off + ranges.back().len) {
      const uint64_t end = ranges.back().off + ranges.back().len;
      if (to <= end) return;
      from = end;
      ranges.back().len = to - ranges.back().off;
    } else {
      ranges.push_back(Range{off, len});
    }
    bytes.insert(bytes.end(), tar + from, tar + to);
  }
};

extern "C" {

// *ranges: n_ranges (off, len) pairs; *bytes: their bytes back to back (free both with lb2emu_free);
// res: members, stop offset, stop reason
int lb2emu_tar_walk(const uint8_t *tar, uint64_t n, uint64_t **ranges, uint64_t *n_ranges, uint8_t **bytes, uint64_t *n_bytes,
                    uint64_t *res) {
  HostIo io;
  io.tar = tar;
  WalkResult r;
  walk(io, tar, n, r);
  *n_ranges = io.ranges.size();
  *ranges = (uint64_t *)malloc(16 * io.ranges.size() + 16);
  memcpy(*ranges, io.ranges.data(), 16 * io.ranges.size());
  *n_bytes = io.bytes.size();
  *bytes = (uint8_t *)malloc(io.bytes.size() + 1);
  memcpy(*bytes, io.bytes.data(), io.bytes.size());
  res[0] = r.members;
  res[1] = r.stop_off;
  res[2] = r.reason;
  return 0;
}

void lb2emu_free(void *p) { free(p); }
}
