// elf_deps.cu -- the dynamic sections of shared objects in device memory behind lb2_elf_deps (api.cu); the parse itself
// is elf_deps.cuh.
//
// One warp per object.  The count pass parses every object and sizes its records and string bytes; the host scans
// the sizes; the write pass parses the objects that came out ST_OK again and writes their records and strings at the
// scanned offsets.  Within a parse the lanes test 32 program headers, dynamic entries or string bytes at a time and a
// ballot finds the first (or last) hit, so a scan of k items costs k / 32 dependent loads.  Objects lie anywhere and
// at any alignment: every field is read byte by byte.
#include "lb2_common.cuh"
#include "elf_deps.cuh"

namespace lb2 {
namespace {
using elfd::Object;
using elfd::Record;

struct WarpLanes {
  uint32_t lane;
  template <class P> __device__ uint64_t first(uint64_t from, uint64_t to, P pred) {
    for (uint64_t b = from; b < to; b += 32) {
      const uint64_t i = b + lane;
      const uint32_t m = __ballot_sync(0xFFFFFFFFu, i < to && pred(i));
      if (m) return b + (__ffs(m) - 1);
    }
    return to;
  }
  template <class P> __device__ uint64_t last(uint64_t from, uint64_t to, P pred) {
    for (uint64_t e = to; e > from; e = e - from > 32 ? e - 32 : from) {
      const uint64_t i = e - 1 - lane;  // lane 0 takes the highest index
      const uint32_t m = __ballot_sync(0xFFFFFFFFu, e - from > lane && pred(i));
      if (m) return e - 1 - (__ffs(m) - 1);
    }
    return to;
  }
  __device__ bool leader() const { return lane == 0; }
  __device__ void copy(uint8_t *dst, const uint8_t *src, uint64_t len) {
    for (uint64_t i = lane; i < len; i += 32) dst[i] = src[i];
    __syncwarp();
  }
};

constexpr int WARPS = 4;

__global__ void __launch_bounds__(32 * WARPS) lb2_elf_deps_count_kernel(const uint64_t *ptrs, const uint64_t *sizes, uint32_t n,
                                                                      Object *obj) {
  const uint32_t i = blockIdx.x * WARPS + threadIdx.x / 32;
  if (i >= n) return;
  WarpLanes lanes{threadIdx.x & 31};
  elfd::Count c;
  uint16_t machine, type;
  const int32_t st = elfd::parse(lanes, reinterpret_cast<const uint8_t *>(ptrs[i]), sizes[i], c, machine, type);
  if (lanes.leader()) {
    const bool ok = st == elfd::ST_OK;
    obj[i] = Object{st, machine, type, 0, ok ? c.n : 0, 0, ok ? c.pool : 0};
  }
}

__global__ void __launch_bounds__(32 * WARPS) lb2_elf_deps_write_kernel(const uint64_t *ptrs, const uint64_t *sizes, uint32_t n,
                                                                      const Object *obj, Record *rec, uint8_t *pool,
                                                                      uint64_t pool_cap) {
  const uint32_t i = blockIdx.x * WARPS + threadIdx.x / 32;
  if (i >= n || obj[i].status != elfd::ST_OK || !obj[i].n_records) return;
  WarpLanes lanes{threadIdx.x & 31};
  const uint64_t end = obj[i].pool_off + obj[i].pool_len;
  elfd::Write w{rec + obj[i].first_record, pool, obj[i].pool_off, obj[i].n_records,
                 end <= pool_cap ? obj[i].pool_len : 0};
  uint16_t machine, type;
  elfd::parse(lanes, reinterpret_cast<const uint8_t *>(ptrs[i]), sizes[i], w, machine, type);
}

}  // namespace

void launch_elf_deps_count(const uint64_t *ptrs, const uint64_t *sizes, uint32_t n, void *obj, cudaStream_t s) {
  if (n) lb2_elf_deps_count_kernel<<<(n + WARPS - 1) / WARPS, 32 * WARPS, 0, s>>>(ptrs, sizes, n, static_cast<Object *>(obj));
}

void launch_elf_deps_write(const uint64_t *ptrs, const uint64_t *sizes, uint32_t n, const void *obj, void *rec, uint8_t *pool,
                           uint64_t pool_cap, cudaStream_t s) {
  if (n)
    lb2_elf_deps_write_kernel<<<(n + WARPS - 1) / WARPS, 32 * WARPS, 0, s>>>(ptrs, sizes, n, static_cast<const Object *>(obj),
                                                                           static_cast<Record *>(rec), pool, pool_cap);
}

}  // namespace lb2
