// api.cu -- C ABI (include/lambdipy_b200.h) over the plan / scan / compaction kernels: the context, the batch core
// that every strip path queues its batches through, the entry points on device-resident arenas, the corpus helpers
// and the host side of the gzip and zip writers and of the gzip reader.  The host-buffer pipelines of lb2_strip_host are in
// strip_host.cu, the tree walker and its streaming engine in strip_tree.cu.
#include "lb2_host.cuh"

#include <cctype>
#include <cstdio>

static thread_local std::string g_create_error;

// NUMA node of the GPU's PCIe root (-1: unknown), where NumaPreferred places the pinned arenas.
static int gpu_numa_node(int device) {
  char bus[64] = {0};
  if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) { cudaGetLastError(); return -1; }
  for (char *c = bus; *c; c++) *c = (char)tolower(*c);
  std::string path = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
  FILE *f = fopen(path.c_str(), "r");
  if (!f) return -1;
  int node = -1;
  if (fscanf(f, "%d", &node) != 1) node = -1;
  fclose(f);
  return node;
}

// Control data of a batch (offsets up; counters, sizes, status, upload ranges down) normally rides on small
// cudaMemcpyAsync calls.  In the host-buffer DMA pipeline those would queue on the copy engines behind 100 MB
// transfers of the neighbouring chunks and stall the host for milliseconds, so there the kernels read the
// offsets through the mapping of the pinned staging buffer and this kernel stores the results into mapped
// pinned memory with ordinary SM stores: no copy engine involved.
__global__ void lb2_zero_ctr_kernel(BatchCounters *ctr) {
  if (threadIdx.x < sizeof(BatchCounters) / 4) reinterpret_cast<uint32_t *>(ctr)[threadIdx.x] = 0;
}
__global__ void __launch_bounds__(256) lb2_publish_kernel(const BatchCounters *ctr, const uint64_t *out_off, const uint64_t *out_size,
                                                          const int32_t *status, const UpRange *ranges, uint32_t n, uint32_t range_cap,
                                                          BatchCounters *h_ctr, uint64_t *h_off, uint64_t *h_size, int32_t *h_status, UpRange *h_ranges) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
  if (t < sizeof(BatchCounters) / 4) reinterpret_cast<uint32_t *>(h_ctr)[t] = reinterpret_cast<const uint32_t *>(ctr)[t];
  for (uint32_t i = t; i <= n; i += stride) h_off[i] = out_off[i];
  for (uint32_t i = t; i < n; i += stride) { h_size[i] = out_size[i]; h_status[i] = status[i]; }
  if (ranges) {
    const uint32_t nr = ctr->n_ranges < range_cap ? ctr->n_ranges : range_cap;
    for (uint32_t i = t; i < nr; i += stride) h_ranges[i] = ranges[i];
  }
}

void ws_free(Workspace &w) {
  cudaFree(w.d_in_off); cudaFree(w.d_in_size); cudaFree(w.d_out_size); cudaFree(w.d_out_off); cudaFree(w.d_status);
  cudaFree(w.d_scratch); cudaFree(w.d_tiles); cudaFree(w.d_ctr);
  if (w.h_stage) cudaFreeHost(w.h_stage);
  if (w.h_res) cudaFreeHost(w.h_res);
  if (w.h_ctr) cudaFreeHost(w.h_ctr);
  cudaFree(w.d_ranges);
  cudaFree(w.d_big);
  if (w.h_ranges) cudaFreeHost(w.h_ranges);
  for (auto &e : w.ev) if (e) cudaEventDestroy(e);
  if (w.done) cudaEventDestroy(w.done);
  w = Workspace();
}

int ws_reserve(lb2_ctx *ctx, Workspace &w, uint32_t n_files, uint64_t n_tiles) {
  if (!w.d_ctr) {
    CK(cudaMalloc(&w.d_ctr, sizeof(BatchCounters)));
    CK(cudaHostAlloc(&w.h_ctr, sizeof(BatchCounters) + 64, cudaHostAllocMapped));
    for (auto &e : w.ev) CK(cudaEventCreate(&e));
    CK(cudaEventCreateWithFlags(&w.done, cudaEventDisableTiming));
  }
  if (n_files > w.cap_files) {
    uint32_t cap = std::max<uint32_t>(n_files, 256u);
    cap = std::max<uint32_t>(cap, w.cap_files + w.cap_files / 2);
    cudaFree(w.d_in_off); cudaFree(w.d_in_size); cudaFree(w.d_out_size); cudaFree(w.d_out_off); cudaFree(w.d_status); cudaFree(w.d_scratch);
    if (w.h_stage) cudaFreeHost(w.h_stage);
    if (w.h_res) cudaFreeHost(w.h_res);
    w.h_stage = nullptr; w.h_res = nullptr;
    w.d_in_off = w.d_in_size = w.d_out_size = w.d_out_off = nullptr; w.d_status = nullptr; w.d_scratch = nullptr;
    w.cap_files = 0;
    CK(cudaMalloc(&w.d_in_off, (cap + 1) * sizeof(uint64_t)));
    CK(cudaMalloc(&w.d_in_size, (cap + 1) * sizeof(uint64_t)));
    CK(cudaMalloc(&w.d_out_size, (cap + 1) * sizeof(uint64_t)));
    CK(cudaMalloc(&w.d_out_off, (cap + 1) * sizeof(uint64_t)));
    CK(cudaMalloc(&w.d_status, (cap + 1) * sizeof(int32_t)));
    CK(cudaMalloc(&w.d_scratch, (uint64_t)cap * SCR_STRIDE));
    CK(cudaHostAlloc(&w.h_stage, (2ull * cap + 2) * sizeof(uint64_t), cudaHostAllocMapped));
    CK(cudaHostAlloc(&w.h_res, (2ull * cap + 2) * sizeof(uint64_t) + (cap + 1ull) * sizeof(int32_t), cudaHostAllocMapped));
    w.cap_files = cap;
  }
  if (n_tiles > w.cap_tiles) CK(regrow(&w.d_tiles, w.cap_tiles, std::max<uint64_t>(n_tiles, w.cap_tiles + w.cap_tiles / 2)));
  return LB2_OK;
}

// Upper bound on the tiles a batch can emit: an extent of l bytes yields at most l / TILE + 2 tiles, a
// file has at most MAX_EXT extents, and re-laid-out files may grow (LOAD alignment padding) -- 1 GB of
// growth per batch is allowed for before the plan kernel reports overflow.
static uint64_t tile_bound(const uint64_t *sizes, uint32_t n) {
  uint64_t t = 65536;
  for (uint32_t i = 0; i < n; i++) t += sizes[i] / TILE_BYTES + 2 * MAX_EXT + 16;
  return t;
}

int enqueue_batch(lb2_ctx *ctx, Workspace &w, const uint8_t *d_in, const uint64_t *h_off, const uint64_t *h_sizes, uint32_t n,
                  uint8_t *d_out, uint64_t out_cap, uint32_t flags, cudaStream_t s, bool compact, bool export_ranges,
                  bool via_mapping) {
  for (uint32_t i = 0; i < n; i++)
    if (h_off[i] & 15) { ctx->err = "input offsets must be multiples of 16"; return LB2_E_ARG; }
  // sizes -> staging (pinned), upload
  std::vector<uint64_t> tmp;
  if (w.in_flight) { ctx->err = "previous batch on this workspace not collected"; return LB2_E_STATE; }
  uint64_t *st_off = nullptr, *st_size = nullptr;
  {
    // need sizes before reserve to bound tiles
    tmp.resize(n);
    for (uint32_t i = 0; i < n; i++) tmp[i] = h_sizes ? h_sizes[i] : (h_off[i + 1] - h_off[i]);
  }
  int rc = ws_reserve(ctx, w, n, tile_bound(tmp.data(), n));
  if (rc) return rc;
  st_off = w.h_stage;
  st_size = w.h_stage + (w.cap_files + 1);
  memcpy(st_off, h_off, (size_t)n * sizeof(uint64_t));
  memcpy(st_size, tmp.data(), (size_t)n * sizeof(uint64_t));
  const uint64_t *k_in_off = w.d_in_off, *k_in_size = w.d_in_size;
  if (via_mapping) {  // no copy-engine traffic for control data (see lb2_publish_kernel)
    void *alias = nullptr;
    CK(cudaHostGetDevicePointer(&alias, w.h_stage, 0));
    k_in_off = static_cast<const uint64_t *>(alias);
    k_in_size = k_in_off + (w.cap_files + 1);
    lb2_zero_ctr_kernel<<<1, 64, 0, s>>>(w.d_ctr);
  } else {
    CK(cudaMemcpyAsync(w.d_in_off, st_off, (size_t)n * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(w.d_in_size, st_size, (size_t)n * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(w.d_ctr, 0, sizeof(BatchCounters), s));
  }
  CK(cudaEventRecord(w.ev[0], s));
  if (export_ranges && w.cap_ranges < 8u * n + 4096u) {
    const uint32_t cap = 8u * std::max<uint32_t>(n, w.cap_files) + 4096u;
    if (w.h_ranges) cudaFreeHost(w.h_ranges);
    w.h_ranges = nullptr; w.cap_ranges = 0;
    CK(cudaHostAlloc(&w.h_ranges, (size_t)cap * sizeof(UpRange), cudaHostAllocMapped));
    CK(regrow(&w.d_ranges, w.cap_ranges, cap));  // sets cap_ranges once both copies exist
  }
  PlanArgs pa;
  pa.in = d_in; pa.in_off = k_in_off; pa.in_size = k_in_size; pa.n_files = n; pa.flags = flags;
  pa.scratch = w.d_scratch; pa.out_size = w.d_out_size; pa.status = w.d_status;
  pa.tiles = w.d_tiles; pa.tile_cap = w.cap_tiles; pa.ctr = w.d_ctr;
  pa.up_ranges = export_ranges ? w.d_ranges : nullptr; pa.up_cap = export_ranges ? w.cap_ranges : 0;
  if (w.cap_big < 8u * n + 4096u) CK(regrow(&w.d_big, w.cap_big, 8u * std::max<uint32_t>(n, w.cap_files) + 4096u));
  pa.big = w.d_big; pa.big_cap = w.cap_big;
  launch_plan(pa, s);
  launch_scan(w.d_out_size, w.d_out_off, n, compact ? out_cap : ~0ull, w.d_ctr, w.d_big, w.cap_big, w.d_tiles, ctx->sm_count * 2, s);
  CK(cudaEventRecord(w.ev[1], s));
  if (compact) {
    CompactArgs ca;
    ca.tiles = w.d_tiles; ca.ctr = w.d_ctr; ca.out_off = w.d_out_off; ca.out = d_out;
    ca.rebase_lo = ca.rebase_len = ca.rebase_delta = 0;
    enqueue_compact(ctx, ca, s);
  }
  CK(cudaEventRecord(w.ev[2], s));
  // results ride behind the kernels into pinned staging; collect_batch only waits for `done`, so a
  // caller may queue the next batch (other workspace, same stream) before collecting this one
  {
    uint64_t *r_off = reinterpret_cast<uint64_t *>(w.h_res), *r_size = r_off + (w.cap_files + 1);
    int32_t *r_status = reinterpret_cast<int32_t *>(r_size + (w.cap_files + 1));
    if (via_mapping) {
      void *a_ctr = nullptr, *a_res = nullptr, *a_rng = nullptr;
      CK(cudaHostGetDevicePointer(&a_ctr, w.h_ctr, 0));
      CK(cudaHostGetDevicePointer(&a_res, w.h_res, 0));
      if (export_ranges) CK(cudaHostGetDevicePointer(&a_rng, w.h_ranges, 0));
      uint64_t *m_off = static_cast<uint64_t *>(a_res), *m_size = m_off + (w.cap_files + 1);
      int32_t *m_status = reinterpret_cast<int32_t *>(m_size + (w.cap_files + 1));
      lb2_publish_kernel<<<std::max(1u, std::min(32u, (n + 255u) / 256u)), 256, 0, s>>>(
          w.d_ctr, w.d_out_off, w.d_out_size, w.d_status, export_ranges ? w.d_ranges : nullptr, n, w.cap_ranges,
          static_cast<BatchCounters *>(a_ctr), m_off, m_size, m_status, static_cast<UpRange *>(a_rng));
    } else {
      CK(cudaMemcpyAsync(w.h_ctr, w.d_ctr, sizeof(BatchCounters), cudaMemcpyDeviceToHost, s));
      if (export_ranges) CK(cudaMemcpyAsync(w.h_ranges, w.d_ranges, (size_t)std::min<uint32_t>(w.cap_ranges, 8u * n + 4096u) * sizeof(UpRange), cudaMemcpyDeviceToHost, s));
      CK(cudaMemcpyAsync(r_off, w.d_out_off, (size_t)(n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
      if (n) {
        CK(cudaMemcpyAsync(r_size, w.d_out_size, (size_t)n * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(r_status, w.d_status, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
      }
    }
    CK(cudaEventRecord(w.done, s));
  }
  CK(cudaGetLastError());
  w.n_files = n;
  w.in_flight = true;
  return LB2_OK;
}

int collect_batch(lb2_ctx *ctx, Workspace &w, uint64_t *h_out_off, uint64_t *h_out_sizes, int32_t *h_status, lb2_stats *stats) {
  if (!w.in_flight) { ctx->err = "no batch in flight"; return LB2_E_STATE; }
  const uint32_t n = w.n_files;
  CK(cudaEventSynchronize(w.done));
  w.in_flight = false;
  const uint64_t *r_off = reinterpret_cast<const uint64_t *>(w.h_res), *r_size = r_off + (w.cap_files + 1);
  const int32_t *r_status = reinterpret_cast<const int32_t *>(r_size + (w.cap_files + 1));
  if (h_out_off) memcpy(h_out_off, r_off, (size_t)(n + 1) * sizeof(uint64_t));
  if (h_out_sizes && n) memcpy(h_out_sizes, r_size, (size_t)n * sizeof(uint64_t));
  if (h_status && n) memcpy(h_status, r_status, (size_t)n * sizeof(int32_t));
  if (stats) {
    const BatchCounters &c = *w.h_ctr;
    memset(stats, 0, sizeof(*stats));
    stats->n_files = n; stats->n_ok = c.n_ok; stats->n_unsupported = c.n_unsupported; stats->overflow = c.overflow;
    stats->in_bytes = c.in_bytes; stats->out_bytes = c.out_bytes; stats->copy_bytes = c.copy_bytes;
    stats->header_bytes = c.header_bytes; stats->n_tiles = c.n_tiles; stats->out_bytes_needed = r_off[n];
    cudaEventElapsedTime(&stats->plan_ms, w.ev[0], w.ev[1]);
    cudaEventElapsedTime(&stats->compact_ms, w.ev[1], w.ev[2]);
  }
  if (w.h_ctr->overflow) { ctx->err = "output arena (or tile buffer) too small for this batch"; return LB2_E_CAPACITY; }
  return LB2_OK;
}

int redo_grown(lb2_ctx *ctx, Workspace &w, const uint8_t *d_in, const uint64_t *h_off, const uint64_t *h_sizes, uint32_t n,
               uint8_t *&d_out, uint64_t &cap_out, uint32_t flags, cudaStream_t s, uint64_t *h_out_off, uint64_t *h_out_sizes,
               int32_t *h_status, lb2_stats *st) {
  const uint64_t need = st->out_bytes_needed + (1u << 20);
  if (cap_out < need) CK(regrow(&d_out, cap_out, need));
  int rc = enqueue_batch(ctx, w, d_in, h_off, h_sizes, n, d_out, cap_out, flags, s, true);
  if (rc) return rc;
  return collect_batch(ctx, w, h_out_off, h_out_sizes, h_status, st);
}

void enqueue_compact(lb2_ctx *ctx, const CompactArgs &ca, cudaStream_t s) {
  if (ctx->use_tma) launch_compact_tma(ca, ctx->sm_count, s);
  else launch_compact(ca, ctx->sm_count * ctx->compact_ctas_per_sm, s);
}

void add_stats(lb2_stats &total, const lb2_stats &st) {
  total.n_ok += st.n_ok; total.n_unsupported += st.n_unsupported; total.in_bytes += st.in_bytes; total.out_bytes += st.out_bytes;
  total.copy_bytes += st.copy_bytes; total.header_bytes += st.header_bytes; total.n_tiles += st.n_tiles;
  total.plan_ms += st.plan_ms; total.compact_ms += st.compact_ms;
}

std::vector<Chunk> split_chunks(const uint64_t *h_in_off, uint32_t n_files, uint64_t max_bytes) {
  std::vector<Chunk> chunks;
  for (uint32_t f = 0; f < n_files;) {
    uint32_t g = f + 1;
    while (g < n_files && h_in_off[g + 1] - h_in_off[f] <= max_bytes) g++;
    chunks.push_back({f, g, h_in_off[f], ((h_in_off[g] - h_in_off[f]) + 255) & ~255ull});
    f = g;
  }
  return chunks;
}

// ============================================================================ C ABI
extern "C" {

const char *lb2_version(void) { return "lambdipy_b200 0.1 (sm_90a; GNU strip 2.42 semantics)"; }

int lb2_ctx_create(int device, lb2_ctx **out) {
  if (!out) return LB2_E_ARG;
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    g_create_error = std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    return LB2_E_NODEVICE;
  }
  if (device < 0 || device >= count) { g_create_error = "device index out of range"; return LB2_E_ARG; }
  lb2_ctx *ctx = new lb2_ctx();
  ctx->device = device;
  if ((e = cudaSetDevice(device)) != cudaSuccess || (e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess) {
    g_create_error = std::string("cuda init: ") + cudaGetErrorString(e);
    delete ctx;
    return LB2_E_CUDA;
  }
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  ctx->sm_count = prop.multiProcessorCount;
  ctx->numa_node = gpu_numa_node(device);
  if (prop.major != 9 || prop.minor != 0) {  // sm_90a code loads on compute capability 9.0 only
    g_create_error = "this library is built for sm_90a (H100) only; device is sm_" + std::to_string(prop.major) + std::to_string(prop.minor);
    cudaStreamDestroy(ctx->stream);
    delete ctx;
    return LB2_E_NODEVICE;
  }
  if (const char *v = getenv("LB2_COMPACT_CTAS_PER_SM")) ctx->compact_ctas_per_sm = std::max(1, atoi(v));
  if (const char *v = getenv("LB2_COMPACT_TMA")) ctx->use_tma = atoi(v);
  *out = ctx;
  return LB2_OK;
}

void lb2_ctx_destroy(lb2_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  ws_free(ctx->ws);
  ws_free(ctx->ws2);
  host_slots_free(ctx->host);
  tree_engine_free(ctx->tree);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

const char *lb2_last_error(const lb2_ctx *ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }
int lb2_sm_count(const lb2_ctx *ctx) { return ctx ? ctx->sm_count : 0; }

void *lb2_dev_alloc(lb2_ctx *ctx, uint64_t bytes) {
  void *p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes ? bytes : 256);
  if (e != cudaSuccess) { if (ctx) ctx->err = std::string("cudaMalloc: ") + cudaGetErrorString(e); return nullptr; }
  return p;
}
void lb2_dev_free(lb2_ctx *, void *p) { if (p) cudaFree(p); }
void *lb2_pinned_alloc(lb2_ctx *ctx, uint64_t bytes) {
  void *p = nullptr;
  NumaPreferred near_gpu(ctx ? ctx->numa_node : -1);
  cudaError_t e = cudaHostAlloc(&p, bytes ? bytes : 256, cudaHostAllocMapped | cudaHostAllocPortable);
  if (e != cudaSuccess) { if (ctx) ctx->err = std::string("cudaHostAlloc: ") + cudaGetErrorString(e); return nullptr; }
  return p;
}
void lb2_pinned_free(lb2_ctx *, void *p) { if (p) cudaFreeHost(p); }
int lb2_memcpy_h2d(lb2_ctx *ctx, void *d, const void *h, uint64_t n) { CK(cudaMemcpy(d, h, n, cudaMemcpyHostToDevice)); return LB2_OK; }
int lb2_memcpy_d2h(lb2_ctx *ctx, void *h, const void *d, uint64_t n) { CK(cudaMemcpy(h, d, n, cudaMemcpyDeviceToHost)); return LB2_OK; }
int lb2_memset_d(lb2_ctx *ctx, void *d, int v, uint64_t n) { CK(cudaMemset(d, v, n)); return LB2_OK; }

int lb2_strip_device_async(lb2_ctx *ctx, const void *d_in, const uint64_t *h_in_off, const uint64_t *h_in_sizes,
                           uint32_t n_files, void *d_out, uint64_t out_capacity, uint32_t flags, void *stream) {
  if (!ctx || !d_in || !h_in_off || !d_out) { if (ctx) ctx->err = "NULL argument"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  if (ctx->async_count >= 2) { ctx->err = "two batches already in flight: collect one with lb2_batch_results first"; return LB2_E_STATE; }
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ctx->stream;
  Workspace &w = ((ctx->async_head + ctx->async_count) & 1) ? ctx->ws2 : ctx->ws;
  int rc = enqueue_batch(ctx, w, static_cast<const uint8_t *>(d_in), h_in_off, h_in_sizes, n_files,
                         static_cast<uint8_t *>(d_out), out_capacity, flags, s, true);
  if (rc == LB2_OK) ctx->async_count++;
  return rc;
}

int lb2_batch_results(lb2_ctx *ctx, uint64_t *h_out_off, uint64_t *h_out_sizes, int32_t *h_status, lb2_stats *stats) {
  if (!ctx) return LB2_E_ARG;
  if (ctx->async_count == 0) { ctx->err = "no batch in flight"; return LB2_E_STATE; }
  Workspace &w = (ctx->async_head & 1) ? ctx->ws2 : ctx->ws;
  ctx->async_head ^= 1;
  ctx->async_count--;
  return collect_batch(ctx, w, h_out_off, h_out_sizes, h_status, stats);
}

int lb2_plan_device(lb2_ctx *ctx, const void *d_in, const uint64_t *h_in_off, const uint64_t *h_in_sizes, uint32_t n_files,
                    uint32_t flags, uint64_t *h_out_sizes, int32_t *h_status, lb2_stats *stats) {
  if (!ctx || !d_in || !h_in_off) { if (ctx) ctx->err = "NULL argument"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  if (ctx->async_count) { ctx->err = "batches of lb2_strip_device_async still in flight"; return LB2_E_STATE; }
  int rc = enqueue_batch(ctx, ctx->ws, static_cast<const uint8_t *>(d_in), h_in_off, h_in_sizes, n_files, nullptr, 0, flags,
                         ctx->stream, false);
  if (rc) return rc;
  return collect_batch(ctx, ctx->ws, nullptr, h_out_sizes, h_status, stats);
}

// ---------------------------------------------------------------------------- shards larger than HBM
// A shard whose input plus output does not fit next to each other in HBM keeps its INPUT resident and
// streams the OUTPUT through a ring of two
// slots: chunk k (consecutive files, <= max_chunk_bytes of arena span) is stripped into slot k % 2 while
// the consumer still holds chunk k-1.  Chunk k+1 is queued on the stream before chunk k is collected, so
// the GPU never waits for the host between chunks.
int lb2_strip_device_chunked(lb2_ctx *ctx, const void *d_in, const uint64_t *h_in_off, const uint64_t *h_in_sizes, uint32_t n_files,
                             void *d_out_ring, uint64_t slot_capacity, uint64_t max_chunk_bytes, uint32_t flags, void *stream,
                             lb2_chunk_fn on_chunk, void *user, uint64_t *h_out_sizes, int32_t *h_status, lb2_stats *total_out) {
  if (!ctx || !d_in || !h_in_off || !d_out_ring || !slot_capacity) { if (ctx) ctx->err = "NULL argument"; return LB2_E_ARG; }
  if (ctx->async_count) { ctx->err = "batches of lb2_strip_device_async still in flight"; return LB2_E_STATE; }
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ctx->stream;
  if (!max_chunk_bytes || max_chunk_bytes > slot_capacity) max_chunk_bytes = slot_capacity;
  const std::vector<Chunk> chunks = split_chunks(h_in_off, n_files, max_chunk_bytes);
  lb2_stats total;
  memset(&total, 0, sizeof total);
  total.n_files = n_files;
  std::vector<uint64_t> coff, csz;
  std::vector<int32_t> cst;
  int rc = LB2_OK;
  auto enqueue = [&](size_t k) -> int {
    const Chunk &c = chunks[k];
    Workspace &w = (k & 1) ? ctx->ws2 : ctx->ws;
    uint8_t *slot = static_cast<uint8_t *>(d_out_ring) + (k & 1) * slot_capacity;
    // offsets stay absolute inside d_in: a chunk is a window of the file list, not a copy
    return enqueue_batch(ctx, w, static_cast<const uint8_t *>(d_in), h_in_off + c.f0, h_in_sizes ? h_in_sizes + c.f0 : nullptr,
                         c.f1 - c.f0, slot, slot_capacity, flags, s, true);
  };
  auto collect = [&](size_t k) -> int {
    const Chunk &c = chunks[k];
    const uint32_t n = c.f1 - c.f0;
    Workspace &w = (k & 1) ? ctx->ws2 : ctx->ws;
    coff.resize(n + 1); csz.resize(n); cst.resize(n);
    lb2_stats st;
    int r = collect_batch(ctx, w, coff.data(), csz.data(), cst.data(), &st);
    if (r) { total.out_bytes_needed = st.out_bytes_needed; total.overflow = 1; return r; }
    if (h_out_sizes) memcpy(h_out_sizes + c.f0, csz.data(), (size_t)n * sizeof(uint64_t));
    if (h_status) memcpy(h_status + c.f0, cst.data(), (size_t)n * sizeof(int32_t));
    add_stats(total, st);
    if (st.out_bytes_needed > total.out_bytes_needed) total.out_bytes_needed = st.out_bytes_needed;
    if (on_chunk) {
      const uint8_t *slot = static_cast<const uint8_t *>(d_out_ring) + (k & 1) * slot_capacity;
      int u = on_chunk(user, (uint32_t)k, c.f0, n, slot, coff.data(), csz.data(), cst.data(), &st);
      if (u) { ctx->err = "chunk consumer returned " + std::to_string(u); return LB2_E_STATE; }
    }
    return LB2_OK;
  };
  for (size_t k = 0; k < chunks.size() && rc == LB2_OK; k++) {
    if (k >= 2) rc = collect(k - 2);           // frees workspace and output slot k % 2
    if (rc == LB2_OK) rc = enqueue(k);
  }
  for (size_t k = chunks.size() >= 2 ? chunks.size() - 2 : 0; k < chunks.size(); k++) {
    Workspace &w = (k & 1) ? ctx->ws2 : ctx->ws;
    if (!w.in_flight) continue;
    int r = collect(k);                         // always drain what was queued
    if (rc == LB2_OK) rc = r;
  }
  if (total_out) *total_out = total;
  return rc;
}

// ---------------------------------------------------------------------------- corpus fill
int lb2_corpus_fill(lb2_ctx *ctx, void *d_arena, const lb2_fill_region *h_regions, uint32_t n_regions, uint64_t seed, void *stream) {
  if (!ctx || !d_arena || (!h_regions && n_regions)) { if (ctx) ctx->err = "NULL argument"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : ctx->stream;
  if (!n_regions) return LB2_OK;
  // split regions into <= 4 MB pieces so the grid balances
  std::vector<lb2_fill_region> pieces;
  const uint64_t P = 4ull << 20;
  for (uint32_t i = 0; i < n_regions; i++)
    for (uint64_t o = 0; o < h_regions[i].len; o += P) pieces.push_back({h_regions[i].offset + o, std::min(P, h_regions[i].len - o)});
  lb2_fill_region *d_regions = nullptr;
  CK(cudaMalloc(&d_regions, pieces.size() * sizeof(lb2_fill_region)));
  CK(cudaMemcpyAsync(d_regions, pieces.data(), pieces.size() * sizeof(lb2_fill_region), cudaMemcpyHostToDevice, s));
  launch_fill(static_cast<uint8_t *>(d_arena), reinterpret_cast<const FillRegion *>(d_regions), (uint32_t)pieces.size(), seed, ctx->sm_count * 8, s);
  CK(cudaStreamSynchronize(s));
  CK(cudaFree(d_regions));
  CK(cudaGetLastError());
  return LB2_OK;
}

int lb2_corpus_scatter(lb2_ctx *ctx, void *d_arena, const void *h_data, uint64_t data_bytes, const uint64_t *h_dst,
                       const uint64_t *h_src, const uint64_t *h_len, uint32_t n) {
  if (!ctx || !d_arena || (n && (!h_data || !h_dst || !h_src || !h_len))) { if (ctx) ctx->err = "NULL argument"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  if (!n) return LB2_OK;
  cudaStream_t s = ctx->stream;
  uint8_t *d_stage = nullptr;
  CK(cudaMalloc(&d_stage, data_bytes + 256));
  CK(cudaMemcpyAsync(d_stage, h_data, data_bytes, cudaMemcpyHostToDevice, s));
  std::vector<Tile> tiles;
  for (uint32_t i = 0; i < n; i++)
    for (uint64_t o = 0; o < h_len[i]; o += TILE_BYTES) {
      Tile t;
      t.src = reinterpret_cast<uint64_t>(d_stage) + h_src[i] + o;
      t.dst_rel = h_dst[i] + o;
      t.len = (uint32_t)std::min<uint64_t>(TILE_BYTES, h_len[i] - o);
      t.file = 0;
      tiles.push_back(t);
    }
  Tile *d_tiles = nullptr;
  BatchCounters *d_ctr = nullptr;
  uint64_t *d_off = nullptr;
  CK(cudaMalloc(&d_tiles, tiles.size() * sizeof(Tile)));
  CK(cudaMalloc(&d_ctr, sizeof(BatchCounters)));
  CK(cudaMalloc(&d_off, sizeof(uint64_t)));
  BatchCounters c;
  memset(&c, 0, sizeof c);
  c.n_tiles = tiles.size();
  uint64_t zero = 0;
  CK(cudaMemcpyAsync(d_tiles, tiles.data(), tiles.size() * sizeof(Tile), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(d_ctr, &c, sizeof c, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(d_off, &zero, sizeof zero, cudaMemcpyHostToDevice, s));
  CompactArgs ca;
  ca.tiles = d_tiles; ca.ctr = d_ctr; ca.out_off = d_off; ca.out = static_cast<uint8_t *>(d_arena);
  ca.rebase_lo = ca.rebase_len = ca.rebase_delta = 0;
  launch_compact(ca, ctx->sm_count * 4, s);
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  cudaFree(d_stage); cudaFree(d_tiles); cudaFree(d_ctr); cudaFree(d_off);
  return LB2_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------- gzip and zip writers
// Device buffers of one piece in flight.  d_in holds GZ_HIST bytes of history in front of the piece: the tail of the
// stream (gzip) or of the file (zip) that the previous piece left open, copied there from GzWriter::d_hist, so the
// first segment's chunks can look back 32 KB across piece boundaries.  The chunk and segment tables are built on the
// host in h_tab and uploaded with the piece.
struct GzSlot {
  uint8_t *d_in = nullptr, *d_chunk_out = nullptr, *d_out = nullptr;
  uint32_t *d_tok = nullptr, *d_meta = nullptr;  // meta: size | mode | crc, n_chunks each
  uint64_t *d_off = nullptr;
  uint8_t *d_tab = nullptr, *h_tab = nullptr;    // GzChunk[n_chunks] then GzSeg[n_segs]
  GzSegResult *d_seg = nullptr, *h_seg = nullptr;  // per-segment results (lb2_zip_segment layout)
  GzResult *d_res = nullptr, *h_res = nullptr;
  uint64_t cap_bytes = 0, cap_tab = 0;
  uint32_t cap_chunks = 0, cap_segs = 0;
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};  // upload | deflate | best | crc | compact |
  cudaEvent_t done = nullptr;
  uint32_t n_segs = 0;
};

struct GzWriter {
  lb2_ctx *ctx = nullptr;
  cudaStream_t stream = nullptr;
  uint8_t *d_hist = nullptr;   // last <= GZ_HIST bytes of the open stream / file
  uint32_t *d_crc = nullptr;   // running CRC-32 of the open stream / file, advanced by each piece's scan kernel
  uint64_t hist_len = 0;
  bool open = false;           // the last piece submitted left a file open (zip)
  uint32_t *d_best = nullptr;  // LB2_DEFLATE_BEST: best_slots workspace slots of BEST_WS_WORDS words, then the claim counter
  uint32_t best_slots = 0;     // 0: default mode
  GzSlot slot[2];
  int head = 0, count = 0;     // pieces in flight, collected in submission order
  bool finished = false;
  lb2_gzip_stats st{};
};
struct lb2_gzip : GzWriter {};
struct lb2_zip : GzWriter {};

static void gz_slot_free(GzSlot &s) {
  cudaFree(s.d_in); cudaFree(s.d_chunk_out); cudaFree(s.d_out); cudaFree(s.d_tok); cudaFree(s.d_meta); cudaFree(s.d_off);
  cudaFree(s.d_tab); cudaFree(s.d_seg); cudaFree(s.d_res);
  if (s.h_tab) cudaFreeHost(s.h_tab);
  if (s.h_seg) cudaFreeHost(s.h_seg);
  if (s.h_res) cudaFreeHost(s.h_res);
  for (auto &e : s.ev) if (e) cudaEventDestroy(e);
  if (s.done) cudaEventDestroy(s.done);
  s = GzSlot();
}

static int gz_slot_reserve(lb2_ctx *ctx, GzSlot &s, uint64_t n, uint32_t n_chunks, uint32_t n_segs) {
  if (!s.d_res) {
    CK(cudaMalloc(&s.d_res, sizeof(GzResult)));
    CK(cudaHostAlloc(&s.h_res, sizeof(GzResult), cudaHostAllocDefault));
    for (auto &e : s.ev) CK(cudaEventCreate(&e));
    CK(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
  }
  if (n > s.cap_bytes || n_chunks > s.cap_chunks) {
    const uint64_t b = std::max(n, s.cap_bytes), c = std::max(n_chunks, s.cap_chunks);
    cudaFree(s.d_in); cudaFree(s.d_chunk_out); cudaFree(s.d_out); cudaFree(s.d_tok); cudaFree(s.d_meta); cudaFree(s.d_off);
    s.d_in = s.d_chunk_out = s.d_out = nullptr; s.d_tok = s.d_meta = nullptr; s.d_off = nullptr;
    s.cap_bytes = 0; s.cap_chunks = 0;
    CK(cudaMalloc(&s.d_in, GZ_HIST + b + 16));
    CK(cudaMalloc(&s.d_chunk_out, b + GZ_OUT_PAD * c + 64));
    CK(cudaMalloc(&s.d_out, b + 17 * c + 16));  // <= 15 bytes of framing per chunk, 2 per segment (segments <= chunks)
    CK(cudaMalloc(&s.d_tok, b * sizeof(uint32_t) + 16));
    CK(cudaMalloc(&s.d_meta, 3 * c * sizeof(uint32_t)));
    CK(cudaMalloc(&s.d_off, c * sizeof(uint64_t)));
    s.cap_bytes = b; s.cap_chunks = (uint32_t)c;
  }
  const uint64_t tab = (uint64_t)n_chunks * sizeof(GzChunk) + (uint64_t)n_segs * sizeof(GzSeg);
  if (tab > s.cap_tab) {
    const uint64_t t = std::max(tab, 2 * s.cap_tab);
    cudaFree(s.d_tab);
    if (s.h_tab) cudaFreeHost(s.h_tab);
    s.d_tab = s.h_tab = nullptr;
    s.cap_tab = 0;
    CK(cudaMalloc(&s.d_tab, t));
    CK(cudaHostAlloc(&s.h_tab, t, cudaHostAllocDefault));
    s.cap_tab = t;
  }
  if (n_segs > s.cap_segs) {
    cudaFree(s.d_seg);
    if (s.h_seg) cudaFreeHost(s.h_seg);
    s.d_seg = s.h_seg = nullptr;
    s.cap_segs = 0;
    CK(cudaMalloc(&s.d_seg, n_segs * sizeof(GzSegResult)));
    CK(cudaHostAlloc(&s.h_seg, n_segs * sizeof(GzSegResult), cudaHostAllocDefault));
    s.cap_segs = n_segs;
  }
  return LB2_OK;
}

static int gz_create(lb2_ctx *ctx, GzWriter *g, uint32_t flags, const char *what) {
  g->ctx = ctx;
  CK(cudaSetDevice(ctx->device));
  cudaError_t e = cudaSuccess;
  if (flags & LB2_DEFLATE_BEST) {  // one workspace slot per CTA the best-mode kernel keeps resident: one per SM
    int sms = 0;
    if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ctx->device)) == cudaSuccess)
      e = cudaMalloc(&g->d_best, (uint64_t)sms * BEST_WS_WORDS * sizeof(uint32_t) + 16);
    g->best_slots = e == cudaSuccess ? (uint32_t)sms : 0;
  }
  if (e != cudaSuccess || (e = cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking)) != cudaSuccess ||
      (e = cudaMalloc(&g->d_hist, GZ_HIST)) != cudaSuccess || (e = cudaMalloc(&g->d_crc, sizeof(uint32_t))) != cudaSuccess ||
      (e = cudaMemsetAsync(g->d_crc, 0, sizeof(uint32_t), g->stream)) != cudaSuccess) {
    ctx->err = std::string(what) + ": " + cudaGetErrorString(e);
    return LB2_E_CUDA;
  }
  return LB2_OK;
}

static void gz_destroy(GzWriter *g) {
  cudaSetDevice(g->ctx->device);
  if (g->stream) cudaStreamSynchronize(g->stream);
  for (auto &s : g->slot) gz_slot_free(s);
  cudaFree(g->d_hist);
  cudaFree(g->d_crc);
  cudaFree(g->d_best);
  if (g->stream) cudaStreamDestroy(g->stream);
}

// Enqueue one piece of n bytes at h_in holding n_segs segments [seg_off[i], seg_off[i] + seg_len[i]) (validated by
// the caller).  cont: segment 0 continues the open stream / file; ends: segment i's file ends in this piece.
static int gz_submit(GzWriter *g, const void *h_in, uint64_t n, const uint64_t *seg_off, const uint64_t *seg_len,
                     uint32_t n_segs, bool cont, bool last_ends) {
  lb2_ctx *ctx = g->ctx;
  CK(cudaSetDevice(ctx->device));
  GzSlot &s = g->slot[(g->head + g->count) & 1];
  uint64_t n_chunks = 0;
  for (uint32_t i = 0; i < n_segs; i++) n_chunks += seg_len[i] ? (seg_len[i] + GZ_CHUNK - 1) / GZ_CHUNK : 1;
  if (n_chunks > UINT32_MAX / 2) { ctx->err = "piece too large"; return LB2_E_ARG; }
  int rc = gz_slot_reserve(ctx, s, n, (uint32_t)n_chunks, n_segs);
  if (rc) return rc;
  GzChunk *chunks = reinterpret_cast<GzChunk *>(s.h_tab);
  GzSeg *segs = reinterpret_cast<GzSeg *>(s.h_tab + n_chunks * sizeof(GzChunk));
  uint32_t c = 0, n_data = 0;
  for (uint32_t i = 0; i < n_segs; i++) {
    const bool ends = i + 1 < n_segs || last_ends;
    const uint64_t before = i == 0 && cont ? g->hist_len : 0;  // bytes of the segment's file in front of it
    segs[i] = GzSeg{seg_off[i], seg_len[i], c, (i == 0 && cont ? GZ_SEG_CONTINUES : 0u) | (ends ? GZ_SEG_ENDS : 0u)};
    uint64_t p = 0;
    do {
      const uint32_t len = (uint32_t)std::min<uint64_t>(GZ_CHUNK, seg_len[i] - p);
      const uint32_t hist = (uint32_t)std::min<uint64_t>(GZ_HIST, before + p);
      chunks[c++] = GzChunk{seg_off[i] + p, len, hist, i, ends && p + len == seg_len[i]};
      n_data += len != 0;
      p += len;
    } while (p < seg_len[i]);
  }
  cudaStream_t st = g->stream;
  GzPieceArgs a;
  a.in = s.d_in + GZ_HIST; a.n = n; a.n_chunks = c; a.n_segs = n_segs;
  a.chunks = reinterpret_cast<const GzChunk *>(s.d_tab);
  a.segs = reinterpret_cast<const GzSeg *>(s.d_tab + n_chunks * sizeof(GzChunk));
  a.tokens = s.d_tok; a.chunk_out = s.d_chunk_out;
  a.chunk_size = s.d_meta; a.chunk_mode = s.d_meta + c; a.chunk_crc = s.d_meta + 2 * c;
  a.chunk_off = s.d_off; a.out = s.d_out; a.crc_state = g->d_crc; a.seg_res = s.d_seg; a.res = s.d_res;
  a.best_ws = g->d_best; a.best_claim = g->d_best ? g->d_best + (uint64_t)g->best_slots * BEST_WS_WORDS : nullptr;
  a.best_slots = g->best_slots;
  CK(cudaEventRecord(s.ev[0], st));
  if (cont && g->hist_len)
    CK(cudaMemcpyAsync(s.d_in + GZ_HIST - g->hist_len, g->d_hist, g->hist_len, cudaMemcpyDeviceToDevice, st));
  if (n) CK(cudaMemcpyAsync(s.d_in + GZ_HIST, h_in, n, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s.d_tab, s.h_tab, n_chunks * sizeof(GzChunk) + n_segs * sizeof(GzSeg), cudaMemcpyHostToDevice, st));
  CK(cudaEventRecord(s.ev[1], st));
  launch_deflate(a, st);
  CK(cudaEventRecord(s.ev[2], st));
  if (g->best_slots) launch_deflate_best(a, st);
  CK(cudaEventRecord(s.ev[3], st));
  launch_crc32(a, st);
  CK(cudaEventRecord(s.ev[4], st));
  launch_gzip_compact(a, st);
  CK(cudaEventRecord(s.ev[5], st));
  CK(cudaMemcpyAsync(s.h_res, s.d_res, sizeof(GzResult), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(s.h_seg, s.d_seg, n_segs * sizeof(GzSegResult), cudaMemcpyDeviceToHost, st));
  CK(cudaEventRecord(s.done, st));
  // history of the next piece: the last <= 32 KB of the file or stream left open, which end with this piece
  uint64_t keep = 0;
  if (!last_ends) {
    const GzSeg &l = segs[n_segs - 1];
    keep = std::min<uint64_t>(GZ_HIST, l.len + (n_segs == 1 && cont ? g->hist_len : 0));
    if (keep) CK(cudaMemcpyAsync(g->d_hist, s.d_in + GZ_HIST + l.start + l.len - keep, keep, cudaMemcpyDeviceToDevice, st));
  }
  CK(cudaGetLastError());
  g->hist_len = keep;
  g->open = !last_ends;
  g->st.n_chunks += n_data;
  g->st.in_bytes += n;
  s.n_segs = n_segs;
  g->count++;
  return LB2_OK;
}

// Wait for the oldest piece and copy its bytes (and, if segs, its per-segment results) out.
static int gz_collect(GzWriter *g, void *h_out, uint64_t out_cap, uint64_t *out_n, GzSegResult *segs) {
  lb2_ctx *ctx = g->ctx;
  CK(cudaSetDevice(ctx->device));
  GzSlot &s = g->slot[g->head];
  uint64_t total = 0;
  if (s.n_segs) {
    CK(cudaEventSynchronize(s.done));
    total = s.h_res->out_bytes;
    *out_n = total;
    if (total > out_cap) { ctx->err = "output buffer too small for this piece (*out_n bytes needed)"; return LB2_E_CAPACITY; }
    if (!h_out) { ctx->err = "NULL argument"; return LB2_E_ARG; }
    const double t0 = now_s();
    if (total) CK(cudaMemcpy(h_out, s.d_out, total, cudaMemcpyDeviceToHost));
    g->st.d2h_ms += (float)((now_s() - t0) * 1e3);
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, s.ev[0], s.ev[1])); g->st.h2d_ms += ms;
    CK(cudaEventElapsedTime(&ms, s.ev[1], s.ev[2])); g->st.deflate_ms += ms;
    CK(cudaEventElapsedTime(&ms, s.ev[2], s.ev[3])); g->st.deflate_ms += ms; g->st.best_ms += ms;
    CK(cudaEventElapsedTime(&ms, s.ev[4], s.ev[5])); g->st.deflate_ms += ms;
    CK(cudaEventElapsedTime(&ms, s.ev[3], s.ev[4])); g->st.crc_ms += ms;
    g->st.crc32 = s.h_res->crc32;
    g->st.n_stored_chunks += s.h_res->n_stored;
    g->st.n_fixed_chunks += s.h_res->n_fixed;
    g->st.n_opt_chunks += s.h_res->n_opt;
    g->st.out_bytes += total;
    if (segs) std::copy(s.h_seg, s.h_seg + s.n_segs, segs);
  }
  *out_n = total;
  s.n_segs = 0;
  g->head ^= 1;
  g->count--;
  return LB2_OK;
}

extern "C" {

int lb2_gzip_create(lb2_ctx *ctx, uint32_t flags, lb2_gzip **out) {
  if (!ctx || !out) { if (ctx) ctx->err = "NULL argument"; return LB2_E_ARG; }
  *out = nullptr;
  if (flags & ~LB2_DEFLATE_BEST) { ctx->err = "lb2_gzip_create: unknown flags"; return LB2_E_ARG; }
  lb2_gzip *g = new lb2_gzip();
  const int rc = gz_create(ctx, g, flags, "lb2_gzip_create");
  if (rc) { lb2_gzip_destroy(g); return rc; }
  *out = g;
  return LB2_OK;
}

void lb2_gzip_destroy(lb2_gzip *g) {
  if (!g) return;
  gz_destroy(g);
  delete g;
}

int lb2_gzip_submit(lb2_gzip *g, const void *h_in, uint64_t n) {
  if (!g) return LB2_E_ARG;
  lb2_ctx *ctx = g->ctx;
  if (!h_in && n) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  if (g->finished) { ctx->err = "lb2_gzip_submit after lb2_gzip_finish"; return LB2_E_STATE; }
  if (g->count >= 2) { ctx->err = "two pieces already in flight: collect one with lb2_gzip_collect first"; return LB2_E_STATE; }
  if (n > (uint64_t)UINT32_MAX * GZ_CHUNK / 2) { ctx->err = "piece too large"; return LB2_E_ARG; }
  if (!n) {  // nothing to deflate: collect returns 0 bytes
    g->slot[(g->head + g->count) & 1].n_segs = 0;
    g->count++;
    return LB2_OK;
  }
  // the piece is one segment of the stream, which continues from the previous piece and stays open
  const uint64_t off = 0;
  return gz_submit(g, h_in, n, &off, &n, 1, true, false);
}

int lb2_gzip_collect(lb2_gzip *g, void *h_out, uint64_t out_cap, uint64_t *out_n) {
  if (!g) return LB2_E_ARG;
  lb2_ctx *ctx = g->ctx;
  if (!out_n) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  if (!g->count) { ctx->err = "no piece in flight"; return LB2_E_STATE; }
  return gz_collect(g, h_out, out_cap, out_n, nullptr);
}

int lb2_gzip_finish(lb2_gzip *g, void *h_out, uint64_t out_cap, uint64_t *out_n, uint32_t *crc32, uint64_t *isize,
                    lb2_gzip_stats *stats) {
  if (!g) return LB2_E_ARG;
  lb2_ctx *ctx = g->ctx;
  if (!h_out || !out_n) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  if (g->count) { ctx->err = "pieces still in flight: collect them first"; return LB2_E_STATE; }
  if (g->finished) { ctx->err = "lb2_gzip_finish called twice"; return LB2_E_STATE; }
  *out_n = 2;
  if (out_cap < 2) { ctx->err = "output buffer too small"; return LB2_E_CAPACITY; }
  // final block: BFINAL 1, fixed Huffman, end-of-block code -- the two bytes zlib ends a flushed stream with
  static_cast<uint8_t *>(h_out)[0] = 0x03;
  static_cast<uint8_t *>(h_out)[1] = 0x00;
  g->finished = true;
  g->st.out_bytes += 2;
  if (crc32) *crc32 = g->st.crc32;
  if (isize) *isize = g->st.in_bytes;
  if (stats) *stats = g->st;
  return LB2_OK;
}

static_assert(sizeof(GzSegResult) == sizeof(lb2_zip_segment), "the scan kernel writes lb2_zip_segment records");

int lb2_zip_create(lb2_ctx *ctx, uint32_t flags, lb2_zip **out) {
  if (!ctx || !out) { if (ctx) ctx->err = "NULL argument"; return LB2_E_ARG; }
  *out = nullptr;
  if (flags & ~LB2_DEFLATE_BEST) { ctx->err = "lb2_zip_create: unknown flags"; return LB2_E_ARG; }
  lb2_zip *z = new lb2_zip();
  const int rc = gz_create(ctx, z, flags, "lb2_zip_create");
  if (rc) { lb2_zip_destroy(z); return rc; }
  *out = z;
  return LB2_OK;
}

void lb2_zip_destroy(lb2_zip *z) {
  if (!z) return;
  gz_destroy(z);
  delete z;
}

int lb2_zip_submit(lb2_zip *z, const void *h_in, uint64_t n, const uint64_t *seg_off, const uint64_t *seg_len, uint32_t n_segs,
                   uint32_t flags) {
  if (!z) return LB2_E_ARG;
  lb2_ctx *ctx = z->ctx;
  if ((!h_in && n) || !seg_off || !seg_len) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  if (flags & ~(LB2_ZIP_CONTINUES | LB2_ZIP_MORE)) { ctx->err = "lb2_zip_submit: unknown flags"; return LB2_E_ARG; }
  if (!n_segs) { ctx->err = "a piece holds at least one segment"; return LB2_E_ARG; }
  if (n > (uint64_t)UINT32_MAX * GZ_CHUNK / 2) { ctx->err = "piece too large"; return LB2_E_ARG; }
  if (z->count >= 2) { ctx->err = "two pieces already in flight: collect one with lb2_zip_collect first"; return LB2_E_STATE; }
  const bool cont = flags & LB2_ZIP_CONTINUES;
  if (cont && !z->open) { ctx->err = "LB2_ZIP_CONTINUES, but the previous piece left no file open"; return LB2_E_STATE; }
  if (!cont && z->open) { ctx->err = "the previous piece's last file is still open: continue it with LB2_ZIP_CONTINUES"; return LB2_E_STATE; }
  if (cont && seg_off[0]) { ctx->err = "a continued file starts the piece: seg_off[0] must be 0"; return LB2_E_ARG; }
  uint64_t end = 0;
  for (uint32_t i = 0; i < n_segs; i++) {
    if ((seg_off[i] & 15) || seg_off[i] < end || seg_off[i] > n || seg_len[i] > n - seg_off[i]) {
      ctx->err = "segment " + std::to_string(i) + " is unaligned, overlaps the one before it or ends past the piece";
      return LB2_E_ARG;
    }
    end = seg_off[i] + seg_len[i];
  }
  return gz_submit(z, h_in, n, seg_off, seg_len, n_segs, cont, !(flags & LB2_ZIP_MORE));
}

int lb2_zip_collect(lb2_zip *z, void *h_out, uint64_t out_cap, uint64_t *out_n, lb2_zip_segment *segs, lb2_gzip_stats *stats) {
  if (!z) return LB2_E_ARG;
  lb2_ctx *ctx = z->ctx;
  if (!out_n || !segs) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  if (!z->count) { ctx->err = "no piece in flight"; return LB2_E_STATE; }
  const int rc = gz_collect(z, h_out, out_cap, out_n, reinterpret_cast<GzSegResult *>(segs));
  if (rc == LB2_OK && stats) *stats = z->st;
  return rc;
}

}  // extern "C"

// ---------------------------------------------------------------------------- gzip reader
// Speculative parallel inflate (inflate_core.cuh, kernels in inflate.cu).  The body is uploaded once; candidate
// search, count rounds (the chain runs here on the host between rounds), decode, resolve and CRC-32 run on the
// reader's stream; the decoded bytes stay on the device until lb2_inflate_read.
#include "inflate_core.cuh"

struct lb2_inflate {
  lb2_ctx *ctx = nullptr;
  cudaStream_t stream = nullptr;
  uint8_t *d_in = nullptr, *d_out = nullptr;
  uint16_t *d_arena = nullptr;
  uint64_t *d_cand = nullptr;
  ifl::SpanJob *d_jobs = nullptr;
  ifl::SpanResult *d_res = nullptr;
  uint32_t *d_chunk_crc = nullptr, *d_crc = nullptr;
  int32_t *d_err = nullptr;
  uint64_t cap_in = 0, cap_cand = 0, cap_jobs = 0, cap_res = 0, cap_arena = 0, cap_out = 0, cap_chunks = 0;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  uint64_t out_n = 0;
  bool have = false;
};

// (re)allocates *p for `need` elements when `cap` is smaller; LB2_E_CAPACITY when the device has no room
template <class T> static int ifl_grow(lb2_ctx *ctx, T **p, uint64_t &cap, uint64_t need) {
  if (need <= cap) return LB2_OK;
  const cudaError_t e = regrow(p, cap, need, 16);
  if (e == cudaErrorMemoryAllocation) {
    cudaGetLastError();
    ctx->err = "lb2_inflate_run: the stream does not fit in device memory";
    return LB2_E_CAPACITY;
  }
  CK(e);
  return LB2_OK;
}

static float ifl_elapsed(lb2_inflate *d) {
  float ms = 0;
  cudaEventElapsedTime(&ms, d->ev[0], d->ev[1]);
  return ms;
}

extern "C" {

int lb2_inflate_create(lb2_ctx *ctx, uint32_t flags, lb2_inflate **out) {
  if (!ctx || !out) { if (ctx) ctx->err = "NULL argument"; return LB2_E_ARG; }
  *out = nullptr;
  if (flags) { ctx->err = "lb2_inflate_create: no flags are defined"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  lb2_inflate *d = new lb2_inflate();
  d->ctx = ctx;
  cudaError_t e;
  if ((e = cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking)) != cudaSuccess ||
      (e = cudaEventCreate(&d->ev[0])) != cudaSuccess || (e = cudaEventCreate(&d->ev[1])) != cudaSuccess ||
      (e = cudaMalloc(&d->d_crc, sizeof(uint32_t))) != cudaSuccess || (e = cudaMalloc(&d->d_err, sizeof(int32_t))) != cudaSuccess) {
    ctx->err = std::string("lb2_inflate_create: ") + cudaGetErrorString(e);
    lb2_inflate_destroy(d);
    return LB2_E_CUDA;
  }
  *out = d;
  return LB2_OK;
}

void lb2_inflate_destroy(lb2_inflate *d) {
  if (!d) return;
  cudaSetDevice(d->ctx->device);
  if (d->stream) cudaStreamSynchronize(d->stream);
  cudaFree(d->d_in); cudaFree(d->d_out); cudaFree(d->d_arena); cudaFree(d->d_cand); cudaFree(d->d_jobs); cudaFree(d->d_res);
  cudaFree(d->d_chunk_crc); cudaFree(d->d_crc); cudaFree(d->d_err);
  for (auto &e : d->ev) if (e) cudaEventDestroy(e);
  if (d->stream) cudaStreamDestroy(d->stream);
  delete d;
}

int lb2_inflate_run(lb2_inflate *d, const void *h_in, uint64_t n, uint64_t *out_n, lb2_inflate_stats *stats) {
  if (!d) return LB2_E_ARG;
  lb2_ctx *ctx = d->ctx;
  if ((!h_in && n) || !out_n) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  d->have = false;
  *out_n = 0;
  lb2_inflate_stats st{};
  uint64_t span = 128 << 10;
  if (const char *v = getenv("LB2_INFLATE_SPAN_KB")) {
    const long kb = atol(v);
    if (kb < 1) { ctx->err = "LB2_INFLATE_SPAN_KB must be a positive number of KB"; return LB2_E_ARG; }
    span = (uint64_t)kb << 10;
  }
  const uint32_t n_spans = n > span ? (uint32_t)((n + span - 1) / span) : 1;
  cudaStream_t s = d->stream;
  int rc;
  if ((rc = ifl_grow(ctx, &d->d_in, d->cap_in, n)) || (rc = ifl_grow(ctx, &d->d_cand, d->cap_cand, n_spans)) ||
      (rc = ifl_grow(ctx, &d->d_jobs, d->cap_jobs, n_spans)) || (rc = ifl_grow(ctx, &d->d_res, d->cap_res, n_spans)))
    return rc;
  // upload
  CK(cudaEventRecord(d->ev[0], s));
  if (n) CK(cudaMemcpyAsync(d->d_in, h_in, n, cudaMemcpyHostToDevice, s));
  CK(cudaEventRecord(d->ev[1], s));
  CK(cudaEventSynchronize(d->ev[1]));
  st.h2d_ms = ifl_elapsed(d);
  // candidates
  std::vector<uint64_t> cand(n_spans, ifl::KEY_NONE);
  CK(cudaEventRecord(d->ev[0], s));
  launch_inflate_find(d->d_in, n, span, n_spans, d->d_cand, s);
  CK(cudaGetLastError());
  CK(cudaEventRecord(d->ev[1], s));
  if (n_spans > 1) CK(cudaMemcpyAsync(cand.data() + 1, d->d_cand + 1, (n_spans - 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  st.find_ms = ifl_elapsed(d);
  // count rounds and chain
  ifl::Chain c;
  c.init(cand.data(), n_spans, span, n, ifl::GIVE_UP_SPANS);
  std::vector<ifl::SpanJob> jobs;
  std::vector<ifl::SpanResult> res;
  while (!c.done && !c.error) {
    const std::vector<uint32_t> p = c.pending();
    jobs.resize(p.size());
    res.resize(p.size());
    for (size_t i = 0; i < p.size(); i++) jobs[i] = c.job[p[i]];
    CK(cudaMemcpyAsync(d->d_jobs, jobs.data(), jobs.size() * sizeof(ifl::SpanJob), cudaMemcpyHostToDevice, s));
    CK(cudaEventRecord(d->ev[0], s));
    launch_inflate_count(d->d_in, n, d->d_jobs, (uint32_t)jobs.size(), d->d_res, s);
    CK(cudaGetLastError());
    CK(cudaEventRecord(d->ev[1], s));
    CK(cudaMemcpyAsync(res.data(), d->d_res, res.size() * sizeof(ifl::SpanResult), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    st.count_ms += ifl_elapsed(d);
    for (size_t i = 0; i < p.size(); i++) c.set_result(p[i], res[i]);
    c.advance();
  }
  st.n_rounds = c.n_rounds;
  st.n_rejected = c.n_rejected;
  st.n_absorbed = c.n_absorbed;
  if (c.error) {
    ctx->err = "lb2_inflate_run: invalid DEFLATE stream (span status " + std::to_string(c.error) + ")";
    if (stats) *stats = st;
    return LB2_E_DATA;
  }
  const uint64_t total = c.layout();
  const uint32_t n_used = (uint32_t)c.job.size();
  st.n_spans = n_used;
  st.in_bytes = c.in_bytes();
  st.out_bytes = total;
  // 2 bytes per output byte for the u16 arena, 1 for the final bytes
  if ((rc = ifl_grow(ctx, &d->d_arena, d->cap_arena, total)) || (rc = ifl_grow(ctx, &d->d_out, d->cap_out, total)) ||
      (rc = ifl_grow(ctx, &d->d_chunk_crc, d->cap_chunks, (total + GZ_CHUNK - 1) / GZ_CHUNK + 1)))
    return rc;
  // decode, resolve, CRC-32
  CK(cudaMemcpyAsync(d->d_jobs, c.job.data(), n_used * sizeof(ifl::SpanJob), cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(d->d_err, 0, sizeof(int32_t), s));
  CK(cudaEventRecord(d->ev[0], s));
  launch_inflate_decode(d->d_in, n, d->d_jobs, n_used, d->d_arena, d->d_err, s);
  CK(cudaGetLastError());
  CK(cudaEventRecord(d->ev[1], s));
  CK(cudaEventSynchronize(d->ev[1]));
  st.decode_ms = ifl_elapsed(d);
  CK(cudaEventRecord(d->ev[0], s));
  launch_inflate_resolve(d->d_arena, d->d_out, d->d_jobs, n_used, d->d_err, s);
  CK(cudaGetLastError());
  CK(cudaEventRecord(d->ev[1], s));
  CK(cudaEventSynchronize(d->ev[1]));
  st.resolve_ms = ifl_elapsed(d);
  CK(cudaEventRecord(d->ev[0], s));
  launch_crc32(d->d_out, total, d->d_chunk_crc, d->d_crc, s);
  CK(cudaGetLastError());
  CK(cudaEventRecord(d->ev[1], s));
  int32_t err = 0;
  CK(cudaMemcpyAsync(&st.crc32, d->d_crc, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&err, d->d_err, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  st.crc_ms = ifl_elapsed(d);
  if (stats) *stats = st;
  if (err) {
    ctx->err = "lb2_inflate_run: invalid DEFLATE stream (decode status " + std::to_string(err) + ")";
    return LB2_E_DATA;
  }
  d->out_n = total;
  d->have = true;
  *out_n = total;
  return LB2_OK;
}

int lb2_inflate_read(lb2_inflate *d, void *h_out, uint64_t cap) {
  if (!d) return LB2_E_ARG;
  lb2_ctx *ctx = d->ctx;
  if (!d->have) { ctx->err = "lb2_inflate_read: no decoded stream (lb2_inflate_run failed or was not called)"; return LB2_E_STATE; }
  if (cap < d->out_n) { ctx->err = "lb2_inflate_read: buffer smaller than the decoded stream"; return LB2_E_CAPACITY; }
  if (!h_out && d->out_n) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  if (d->out_n) CK(cudaMemcpy(h_out, d->d_out, d->out_n, cudaMemcpyDeviceToHost));
  return LB2_OK;
}

}  // extern "C"
