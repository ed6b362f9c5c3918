// lb2_host.cuh -- host-side state and helpers shared by api.cu (context, batch core, device-resident entry points,
// corpus, gzip), strip_host.cu (lb2_strip_host) and strip_tree.cu (lb2_strip_tree).  Internal: not installed.
#pragma once
#include "lb2_common.cuh"
#include "../../include/lambdipy_b200.h"

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include <sys/syscall.h>
#include <unistd.h>

using namespace lb2;

// Device workspace of one batch in flight.
struct Workspace {
  uint64_t *d_in_off = nullptr, *d_in_size = nullptr, *d_out_size = nullptr, *d_out_off = nullptr;
  int32_t *d_status = nullptr;
  uint8_t *d_scratch = nullptr;
  Tile *d_tiles = nullptr;
  BatchCounters *d_ctr = nullptr;
  UpRange *d_ranges = nullptr, *h_ranges = nullptr;  // host-buffer pipeline: input ranges to upload (pinned copy)
  BigExt *d_big = nullptr;      // extents whose tiles the scan launch's extra CTAs write
  uint32_t cap_big = 0;
  uint32_t cap_ranges = 0;
  uint64_t *h_stage = nullptr;  // pinned: 2*(n+1) offsets/sizes up
  uint8_t *h_res = nullptr;     // pinned: out_off[n+1] | out_size[n] | status[n] down (queued behind the kernels)
  BatchCounters *h_ctr = nullptr;
  cudaEvent_t done = nullptr;   // recorded behind the last result copy: collect waits on this, not on the stream
  uint32_t cap_files = 0;
  uint64_t cap_tiles = 0;
  cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
  // last batch
  uint32_t n_files = 0;
  bool in_flight = false;
};

struct HostSlots;   // strip_host.cu: the three slots of the staged and copy-engine host pipelines
struct TreeEngine;  // strip_tree.cu: pinned slot ring, I/O worker streams, HBM batch buffers
void host_slots_free(HostSlots *h);
void tree_engine_free(TreeEngine *e);

struct lb2_ctx {
  int device = 0;
  int numa_node = -1;          // NUMA node of the GPU's PCIe root (-1: unknown / single node)
  int sm_count = 0;
  cudaStream_t stream = nullptr;
  Workspace ws;               // lb2_strip_device_async / lb2_plan_device / even chunks of lb2_strip_device_chunked
  Workspace ws2;              // odd chunks (chunk k+1 is queued before chunk k is collected)
  int async_head = 0, async_count = 0;  // lb2_strip_device_async: up to two batches in flight (ws, ws2), collected in order
  std::string err;
  int compact_ctas_per_sm = 4;
  int use_tma = 1;             // bulk-copy engine kernel; LB2_COMPACT_TMA=0 selects the LSU kernel
  HostSlots *host = nullptr;   // lb2_strip_host, created on first use
  TreeEngine *tree = nullptr;  // lb2_strip_tree, created on first use
};

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) {                                                                       \
      ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_);                               \
      return LB2_E_CUDA;                                                                           \
    }                                                                                              \
  } while (0)

inline double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

inline uint64_t env_u64(const char *name, uint64_t dflt) {
  const char *v = getenv(name);
  return v ? strtoull(v, nullptr, 10) : dflt;
}

// Pinned host arenas are placed on the NUMA node the GPU hangs off: the compaction kernel of the zero-copy
// host path reads and writes them over PCIe, and a remote-socket arena puts that traffic on the
// inter-socket link as well.
// The policy is set only around the allocation (MPOL_PREFERRED: falls back to other nodes when full).
struct NumaPreferred {
  bool active = false;
  explicit NumaPreferred(int node) {
    const char *v = getenv("LB2_NUMA");
    if (node < 0 || node >= 1024 || (v && atoi(v) == 0)) return;
    unsigned long mask[16] = {0};
    mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
    active = syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, mask, sizeof(mask) * 8 + 1) == 0;
  }
  ~NumaPreferred() { if (active) syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0); }
};

// Replaces the device buffer *p by a new one of `count` elements (plus `pad` bytes) and records `count` in `cap`.
// The old contents are dropped.  On failure *p is null, `cap` is 0 and the error is returned for the caller to report.
template <class T, class C> inline cudaError_t regrow(T **p, C &cap, uint64_t count, uint64_t pad = 0) {
  cudaFree(*p);
  *p = nullptr;
  cap = 0;
  const cudaError_t e = cudaMalloc(p, count * sizeof(T) + pad);
  if (e == cudaSuccess) cap = (C)count;
  return e;
}

// ---- batch core (api.cu)
void ws_free(Workspace &w);
int ws_reserve(lb2_ctx *ctx, Workspace &w, uint32_t n_files, uint64_t n_tiles);
// Enqueue plan -> scan -> (compact) for one batch on `s`.  h_off/h_sizes are host arrays.
int enqueue_batch(lb2_ctx *ctx, Workspace &w, const uint8_t *d_in, const uint64_t *h_off, const uint64_t *h_sizes, uint32_t n,
                  uint8_t *d_out, uint64_t out_cap, uint32_t flags, cudaStream_t s, bool compact, bool export_ranges = false,
                  bool via_mapping = false);
int collect_batch(lb2_ctx *ctx, Workspace &w, uint64_t *h_out_off, uint64_t *h_out_sizes, int32_t *h_status, lb2_stats *stats);
// After a batch returned LB2_E_CAPACITY (*st holds what it needed): grows *d_out to that plus 1 MB when it is
// smaller -- re-laid-out files can grow -- and strips the batch again, waiting for the result.
int redo_grown(lb2_ctx *ctx, Workspace &w, const uint8_t *d_in, const uint64_t *h_off, const uint64_t *h_sizes, uint32_t n,
               uint8_t *&d_out, uint64_t &cap_out, uint32_t flags, cudaStream_t s, uint64_t *h_out_off, uint64_t *h_out_sizes,
               int32_t *h_status, lb2_stats *st);
// The compaction kernel the context selects (LB2_COMPACT_TMA, LB2_COMPACT_CTAS_PER_SM).
void enqueue_compact(lb2_ctx *ctx, const CompactArgs &ca, cudaStream_t s);
// Adds one batch's counters and kernel times into `total` (n_files and out_bytes_needed are the caller's).
void add_stats(lb2_stats &total, const lb2_stats &st);

// Consecutive files, <= max_bytes of arena span each (a bigger file stands alone).  in_base is the first file's
// offset, in_span the chunk's span rounded up to 256 bytes.
struct Chunk { uint32_t f0, f1; uint64_t in_base, in_span; };
std::vector<Chunk> split_chunks(const uint64_t *h_in_off, uint32_t n_files, uint64_t max_bytes);
