// compact_tma.cu -- compaction through the bulk-copy (TMA) engine: cp.async.bulk global->shared
// signalled on an mbarrier, then cp.async.bulk shared->global, 16 KB stages in a shared-memory
// ring.  No registers and no LSU instructions touch the payload; one producer lane and one storer
// lane per CTA drive the engine, the remaining warps take what the engine cannot: heads/tails of
// < 16 bytes, tiles whose source and destination are not congruent mod 16, zero fills.
//
// One persistent CTA per SM (grid = SM count); tiles are claimed dynamically.  SASS: UBLKCP.
#include "lb2_common.cuh"
#include "copy_device.cuh"

namespace lb2 {

constexpr int TMA_STAGES = 12;           // 12 x 16 KB = 192 KB of the 227 KB shared memory
constexpr int TMA_THREADS = 256;         // warp 0: producer, warp 1: storer, warps 2..7: helpers
constexpr uint32_t TMA_MIN_BODY = 2048;  // smaller aligned bodies go through the LSU path
constexpr int TMA_STORES_IN_FLIGHT = 6;  // bulk stores allowed to be still reading shared memory

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void *gdst, const void *smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
               :: "l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(N) : "memory");
}

// How a tile splits between the engine (16-byte aligned body) and the LSU helpers (head, tail).
struct BulkSplit { uint32_t head, body; };
__device__ __forceinline__ BulkSplit bulk_split(const TileView &v) {
  BulkSplit s{0, 0};
  if (!v.src) return s;
  if (((reinterpret_cast<uintptr_t>(v.src) ^ reinterpret_cast<uintptr_t>(v.dst)) & 15) != 0) return s;
  uint32_t head = (uint32_t)((16 - (reinterpret_cast<uintptr_t>(v.dst) & 15)) & 15);
  if (head >= v.len) return s;
  uint32_t body = (v.len - head) & ~15u;
  if (body < TMA_MIN_BODY) return s;
  s.head = head; s.body = body;
  return s;
}

// Work distribution is DYNAMIC: two device-wide claim counters in BatchCounters (zeroed with the rest
// of the struct when the batch is enqueued).  `claim_bulk` feeds the producer warps, 32 tiles per claim;
// `claim_help` feeds the helper warps, 32 tiles per claim.  Every tile is therefore visited twice, once
// per role, by whichever CTA gets there first -- a CTA that starts late or shares its SM with a foreign
// kernel (an NCCL collective on another stream) simply claims less, instead of stretching the kernel by
// its whole static share.
//
// Inside a CTA the producer lane is the only one that sees tile descriptors of engine tiles: it posts
// {destination, bytes} of each stage next to the stage, the storer lane picks them up after the full
// barrier (mbarrier arrive = release, try_wait = acquire), a zero-byte stage is the end marker.
__global__ void __launch_bounds__(TMA_THREADS, 1) lb2_compact_tma_kernel(CompactArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ uint64_t full_bar[TMA_STAGES], empty_bar[TMA_STAGES];
  __shared__ uint64_t stage_dst[TMA_STAGES];
  __shared__ uint32_t stage_len[TMA_STAGES];
  if (a.ctr->overflow) return;
  const unsigned long long n_tiles = a.ctr->n_tiles;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < TMA_STAGES; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ---- producer warp: claim 32 tiles (one descriptor per lane, one round trip to L2 for the whole
    //      batch), hand the engine tiles to lane 0 by shuffle, which queues the bulk loads running up to
    //      TMA_STAGES tiles ahead of the stores.  The claim of the NEXT batch is issued before the
    //      current one is worked off, so its atomic round trip is hidden.
    uint32_t it = 0;
    unsigned long long base = 0, next = 0;
    if (lane == 0) base = atomicAdd(&a.ctr->claim_bulk, 32ull);
    base = __shfl_sync(0xffffffffu, base, 0);
    while (base < n_tiles) {
      if (lane == 0) next = atomicAdd(&a.ctr->claim_bulk, 32ull);
      const unsigned long long t = base + (unsigned long long)lane;
      uint64_t src = 0, dst = 0;
      uint32_t body = 0;
      if (t < n_tiles) {
        const TileView v = load_tile(a, t);
        const BulkSplit sp = bulk_split(v);
        body = sp.body;
        src = reinterpret_cast<uint64_t>(v.src) + sp.head;
        dst = reinterpret_cast<uint64_t>(v.dst) + sp.head;
      }
      unsigned todo = __ballot_sync(0xffffffffu, body != 0);
      while (todo) {
        const int l = __ffs(todo) - 1;
        todo &= todo - 1;
        const uint64_t s_ = __shfl_sync(0xffffffffu, src, l), d_ = __shfl_sync(0xffffffffu, dst, l);
        const uint32_t b_ = __shfl_sync(0xffffffffu, body, l);
        if (lane == 0) {
          const uint32_t st = it % TMA_STAGES, round = it / TMA_STAGES;
          if (round > 0) mbar_wait(&empty_bar[st], (round - 1) & 1);
          stage_dst[st] = d_;
          stage_len[st] = b_;
          mbar_expect_tx(&full_bar[st], b_);
          bulk_g2s(smem + (size_t)st * TILE_BYTES, reinterpret_cast<const void *>(s_), b_, &full_bar[st]);
        }
        it++;
      }
      base = __shfl_sync(0xffffffffu, next, 0);
    }
    if (lane == 0) {  // end marker: a stage of zero bytes
      const uint32_t st = it % TMA_STAGES, round = it / TMA_STAGES;
      if (round > 0) mbar_wait(&empty_bar[st], (round - 1) & 1);
      stage_len[st] = 0;
      mbar_arrive(&full_bar[st]);
    }
  } else if (warp == 1) {
    // ---- storer lane: as a stage lands queue its bulk store; release the stage whose store has
    //      finished reading shared memory
    if (lane == 0) {
      for (uint32_t it = 0;; it++) {
        const uint32_t st = it % TMA_STAGES, round = it / TMA_STAGES;
        mbar_wait(&full_bar[st], round & 1);
        const uint32_t b_ = stage_len[st];
        if (b_ == 0) break;
        bulk_s2g(reinterpret_cast<void *>(stage_dst[st]), smem + (size_t)st * TILE_BYTES, b_);
        bulk_commit();
        if (it >= (uint32_t)TMA_STORES_IN_FLIGHT) {
          bulk_wait_read<TMA_STORES_IN_FLIGHT>();
          mbar_arrive(&empty_bar[(it - TMA_STORES_IN_FLIGHT) % TMA_STAGES]);
        }
      }
      bulk_wait_read<0>();
      asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // stores performed before the CTA exits
    }
  } else {
    // ---- helpers: heads/tails of engine tiles, and every tile the engine does not take.  One
    //      descriptor per lane per claim; only tiles with LSU work cost more than that.
    for (;;) {
      unsigned long long base = 0;
      if (lane == 0) base = atomicAdd(&a.ctr->claim_help, 32ull);
      base = __shfl_sync(0xffffffffu, base, 0);
      if (base >= n_tiles) break;
      const unsigned long long t = base + (unsigned long long)lane;
      uint64_t src = 0, dst = 0;
      uint32_t len = 0, head = 0, body = 0;
      bool work = false;
      if (t < n_tiles) {
        const TileView v = load_tile(a, t);
        const BulkSplit sp = bulk_split(v);
        src = reinterpret_cast<uint64_t>(v.src); dst = reinterpret_cast<uint64_t>(v.dst);
        len = v.len; head = sp.head; body = sp.body;
        work = body ? (head != 0 || head + body != len) : len != 0;
      }
      unsigned todo = __ballot_sync(0xffffffffu, work);
      while (todo) {
        const int l = __ffs(todo) - 1;
        todo &= todo - 1;
        const uint8_t *s_ = reinterpret_cast<const uint8_t *>(__shfl_sync(0xffffffffu, src, l));
        uint8_t *d_ = reinterpret_cast<uint8_t *>(__shfl_sync(0xffffffffu, dst, l));
        const uint32_t len_ = __shfl_sync(0xffffffffu, len, l), head_ = __shfl_sync(0xffffffffu, head, l),
                       body_ = __shfl_sync(0xffffffffu, body, l);
        if (body_) {
          if (lane < (int)head_) d_[lane] = __ldg(s_ + lane);
          const uint32_t done = head_ + body_, tail = len_ - done;
          if (lane < (int)tail) d_[done + lane] = __ldg(s_ + done + lane);
        } else if (s_) {
          warp_copy_tile(s_, d_, len_, lane);
        } else {
          warp_zero_tile(d_, len_, lane);
        }
      }
    }
  }
}

// The 192 KB dynamic shared-memory opt-in is a per-device function attribute: set it once for every
// device this process launches on (several contexts on different GPUs may live in one process).
void launch_compact_tma(const CompactArgs &a, int grid, cudaStream_t s) {
  static bool configured[64] = {};
  const size_t smem = (size_t)TMA_STAGES * TILE_BYTES;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !configured[dev]) {
    cudaFuncSetAttribute(lb2_compact_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (dev >= 0 && dev < 64) configured[dev] = true;
  }
  lb2_compact_tma_kernel<<<grid, TMA_THREADS, smem, s>>>(a);
}

}  // namespace lb2
