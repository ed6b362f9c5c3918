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
int lb2_memcpy_d2d(lb2_ctx *ctx, void *d, const void *s, uint64_t n) {
  if (!ctx) return LB2_E_ARG;
  if ((!d || !s) && n) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  if (!n) return LB2_OK;
  CK(cudaMemcpy(d, s, n, cudaMemcpyDeviceToDevice));
  CK(cudaStreamSynchronize(0));  // a device-to-device cudaMemcpy may return before the copy is done
  return LB2_OK;
}

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
  GzGatherTile *d_gat = nullptr, *h_gat = nullptr;  // lb2_zip_submit_device: the tiles that lay the piece out in d_in
  uint64_t cap_bytes = 0, cap_tab = 0, cap_gat = 0;
  uint32_t cap_chunks = 0, cap_segs = 0;
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};  // upload | deflate | best | crc | compact |
  cudaEvent_t done = nullptr;
  uint32_t n_segs = 0;
  uint32_t n_chunks = 0;
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
  int sizes_slot = -1;         // the slot of the piece collected last while its chunk sizes are still in d_meta
  uint32_t sizes_n = 0;        // its chunk count
};
struct lb2_gzip : GzWriter {};
struct lb2_zip : GzWriter {};

static void gz_slot_free(GzSlot &s) {
  cudaFree(s.d_in); cudaFree(s.d_chunk_out); cudaFree(s.d_out); cudaFree(s.d_tok); cudaFree(s.d_meta); cudaFree(s.d_off);
  cudaFree(s.d_tab); cudaFree(s.d_seg); cudaFree(s.d_res); cudaFree(s.d_gat);
  if (s.h_tab) cudaFreeHost(s.h_tab);
  if (s.h_gat) cudaFreeHost(s.h_gat);
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

// Enqueue one piece of n bytes holding n_segs segments [seg_off[i], seg_off[i] + seg_len[i]) (validated by the
// caller).  The piece is uploaded from h_in, or, when d_src is given, gathered on the device: source j is d_src[j].len
// bytes at d_src[j].d_ptr, laid out at src_dst[j] of the piece and, with pad, followed by zeros up to the next multiple
// of 16 (the zip writer's segments: one source each).  cont: segment 0 continues the open stream / file; ends: segment
// i's file ends in this piece.
static int gz_submit(GzWriter *g, const void *h_in, const lb2_zip_source *d_src, uint32_t n_src, const uint64_t *src_dst,
                     bool pad, uint64_t n, const uint64_t *seg_off, const uint64_t *seg_len, uint32_t n_segs, bool cont,
                     bool last_ends) {
  lb2_ctx *ctx = g->ctx;
  CK(cudaSetDevice(ctx->device));
  const int slot = (g->head + g->count) & 1;
  GzSlot &s = g->slot[slot];
  if (g->sizes_slot == slot) g->sizes_slot = -1;
  uint64_t n_chunks = 0;
  for (uint32_t i = 0; i < n_segs; i++) n_chunks += seg_len[i] ? (seg_len[i] + GZ_CHUNK - 1) / GZ_CHUNK : 1;
  if (n_chunks > UINT32_MAX / 2) { ctx->err = "piece too large"; return LB2_E_ARG; }
  int rc = gz_slot_reserve(ctx, s, n, (uint32_t)n_chunks, n_segs);
  if (rc) return rc;
  uint64_t n_tiles = 0;
  if (d_src) {
    for (uint32_t i = 0; i < n_src; i++) n_tiles += (d_src[i].len + GZ_GATHER_TILE - 1) / GZ_GATHER_TILE;
    if (n_tiles > s.cap_gat) {
      const uint64_t t = std::max(n_tiles, 2 * s.cap_gat);
      cudaFree(s.d_gat);
      if (s.h_gat) cudaFreeHost(s.h_gat);
      s.d_gat = s.h_gat = nullptr;
      s.cap_gat = 0;
      CK(cudaMalloc(&s.d_gat, t * sizeof(GzGatherTile)));
      CK(cudaHostAlloc(&s.h_gat, t * sizeof(GzGatherTile), cudaHostAllocDefault));
      s.cap_gat = t;
    }
    GzGatherTile *tile = s.h_gat;
    for (uint32_t i = 0; i < n_src; i++)
      for (uint64_t p = 0; p < d_src[i].len; p += GZ_GATHER_TILE) {
        const uint32_t len = (uint32_t)std::min<uint64_t>(GZ_GATHER_TILE, d_src[i].len - p);
        const uint64_t end = src_dst[i] + p + len;
        *tile++ = GzGatherTile{static_cast<const uint8_t *>(d_src[i].d_ptr) + p, src_dst[i] + p, len,
                               pad && p + len == d_src[i].len ? (uint32_t)(-end & 15) : 0u};
      }
  }
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
  if (d_src) {
    if (n_tiles) CK(cudaMemcpyAsync(s.d_gat, s.h_gat, n_tiles * sizeof(GzGatherTile), cudaMemcpyHostToDevice, st));
    launch_zip_gather(s.d_gat, (uint32_t)n_tiles, s.d_in + GZ_HIST, st);
  } else if (n) {
    CK(cudaMemcpyAsync(s.d_in + GZ_HIST, h_in, n, cudaMemcpyHostToDevice, st));
  }
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
  s.n_chunks = c;
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
  g->sizes_slot = g->head;
  g->sizes_n = s.n_segs ? s.n_chunks : 0;
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
  return gz_submit(g, h_in, nullptr, 0, nullptr, false, n, &off, &n, 1, true, false);
}

int lb2_gzip_submit_device(lb2_gzip *g, const lb2_zip_source *src, uint32_t n_segs) {
  if (!g) return LB2_E_ARG;
  lb2_ctx *ctx = g->ctx;
  if (!src && n_segs) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  if (g->finished) { ctx->err = "lb2_gzip_submit_device after lb2_gzip_finish"; return LB2_E_STATE; }
  if (g->count >= 2) { ctx->err = "two pieces already in flight: collect one with lb2_gzip_collect first"; return LB2_E_STATE; }
  std::vector<uint64_t> dst(n_segs);
  uint64_t n = 0;  // the piece: the sources back to back
  for (uint32_t i = 0; i < n_segs; i++) {
    if (!src[i].d_ptr && src[i].len) { ctx->err = "segment " + std::to_string(i) + ": NULL source"; return LB2_E_ARG; }
    dst[i] = n;
    if (src[i].len > (uint64_t)UINT32_MAX * GZ_CHUNK / 2 - n) { ctx->err = "piece too large"; return LB2_E_ARG; }
    n += src[i].len;
  }
  if (!n) {
    g->slot[(g->head + g->count) & 1].n_segs = 0;
    g->count++;
    return LB2_OK;
  }
  const uint64_t off = 0;
  return gz_submit(g, nullptr, src, n_segs, dst.data(), false, n, &off, &n, 1, true, false);
}

int lb2_gzip_collect(lb2_gzip *g, void *h_out, uint64_t out_cap, uint64_t *out_n) {
  if (!g) return LB2_E_ARG;
  lb2_ctx *ctx = g->ctx;
  if (!out_n) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  if (!g->count) { ctx->err = "no piece in flight"; return LB2_E_STATE; }
  return gz_collect(g, h_out, out_cap, out_n, nullptr);
}

int lb2_gzip_chunk_sizes(lb2_gzip *g, uint32_t *sizes, uint32_t cap, uint32_t *n_chunks) {
  if (!g) return LB2_E_ARG;
  lb2_ctx *ctx = g->ctx;
  if (!n_chunks) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  *n_chunks = 0;
  if (g->sizes_slot < 0) { ctx->err = "lb2_gzip_chunk_sizes: no piece collected since the last submit into its slot"; return LB2_E_STATE; }
  *n_chunks = g->sizes_n;
  if (cap < g->sizes_n) { ctx->err = "lb2_gzip_chunk_sizes: buffer smaller than the piece's chunk count"; return LB2_E_CAPACITY; }
  if (!sizes && g->sizes_n) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  if (g->sizes_n) CK(cudaMemcpy(sizes, g->slot[g->sizes_slot].d_meta, g->sizes_n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  return LB2_OK;
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

// the checks lb2_zip_submit and lb2_zip_submit_device share, made before the segments are looked at
static int zip_submit_checks(lb2_zip *z, uint32_t n_segs, uint32_t flags) {
  lb2_ctx *ctx = z->ctx;
  if (flags & ~(LB2_ZIP_CONTINUES | LB2_ZIP_MORE)) { ctx->err = "lb2_zip_submit: unknown flags"; return LB2_E_ARG; }
  if (!n_segs) { ctx->err = "a piece holds at least one segment"; return LB2_E_ARG; }
  if (z->count >= 2) { ctx->err = "two pieces already in flight: collect one with lb2_zip_collect first"; return LB2_E_STATE; }
  const bool cont = flags & LB2_ZIP_CONTINUES;
  if (cont && !z->open) { ctx->err = "LB2_ZIP_CONTINUES, but the previous piece left no file open"; return LB2_E_STATE; }
  if (!cont && z->open) { ctx->err = "the previous piece's last file is still open: continue it with LB2_ZIP_CONTINUES"; return LB2_E_STATE; }
  return LB2_OK;
}

int lb2_zip_submit(lb2_zip *z, const void *h_in, uint64_t n, const uint64_t *seg_off, const uint64_t *seg_len, uint32_t n_segs,
                   uint32_t flags) {
  if (!z) return LB2_E_ARG;
  lb2_ctx *ctx = z->ctx;
  if ((!h_in && n) || !seg_off || !seg_len) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  if (n > (uint64_t)UINT32_MAX * GZ_CHUNK / 2) { ctx->err = "piece too large"; return LB2_E_ARG; }
  const int rc = zip_submit_checks(z, n_segs, flags);
  if (rc) return rc;
  const bool cont = flags & LB2_ZIP_CONTINUES;
  if (cont && seg_off[0]) { ctx->err = "a continued file starts the piece: seg_off[0] must be 0"; return LB2_E_ARG; }
  uint64_t end = 0;
  for (uint32_t i = 0; i < n_segs; i++) {
    if ((seg_off[i] & 15) || seg_off[i] < end || seg_off[i] > n || seg_len[i] > n - seg_off[i]) {
      ctx->err = "segment " + std::to_string(i) + " is unaligned, overlaps the one before it or ends past the piece";
      return LB2_E_ARG;
    }
    end = seg_off[i] + seg_len[i];
  }
  return gz_submit(z, h_in, nullptr, 0, nullptr, false, n, seg_off, seg_len, n_segs, cont, !(flags & LB2_ZIP_MORE));
}

int lb2_zip_submit_device(lb2_zip *z, const lb2_zip_source *src, uint32_t n_segs, uint32_t flags) {
  if (!z) return LB2_E_ARG;
  lb2_ctx *ctx = z->ctx;
  if (!src) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  const int rc = zip_submit_checks(z, n_segs, flags);
  if (rc) return rc;
  std::vector<uint64_t> off(n_segs), len(n_segs);
  uint64_t n = 0;  // the piece: every segment at the next multiple of 16
  for (uint32_t i = 0; i < n_segs; i++) {
    if (!src[i].d_ptr && src[i].len) { ctx->err = "segment " + std::to_string(i) + ": NULL source"; return LB2_E_ARG; }
    off[i] = (n + 15) & ~15ull;
    len[i] = src[i].len;
    if (len[i] > (uint64_t)UINT32_MAX * GZ_CHUNK / 2 - off[i]) { ctx->err = "piece too large"; return LB2_E_ARG; }
    n = off[i] + len[i];
  }
  return gz_submit(z, nullptr, src, n_segs, off.data(), true, n, off.data(), len.data(), n_segs, flags & LB2_ZIP_CONTINUES,
                   !(flags & LB2_ZIP_MORE));
}

int lb2_zip_chunk_sizes(lb2_zip *z, uint32_t *sizes, uint32_t cap, uint32_t *n_chunks) {
  return lb2_gzip_chunk_sizes(reinterpret_cast<lb2_gzip *>(static_cast<GzWriter *>(z)), sizes, cap, n_chunks);
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
  ifl::FindJob *d_find = nullptr;
  ifl::SpanJob *d_jobs = nullptr;
  ifl::SpanResult *d_res = nullptr;
  uint32_t *d_chunk_crc = nullptr, *d_crc = nullptr, *d_first = nullptr;
  int32_t *d_err = nullptr;
  uint64_t cap_in = 0, cap_cand = 0, cap_find = 0, cap_jobs = 0, cap_res = 0, cap_arena = 0, cap_out = 0, cap_chunks = 0;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  uint64_t out_n = 0;
  bool have = false;
};

// (re)allocates *p for `need` elements when `cap` is smaller; LB2_E_CAPACITY when the device has no room
template <class T> static int ifl_grow(lb2_ctx *ctx, T **p, uint64_t &cap, uint64_t need,
                                       const char *what = "lb2_inflate_run: the stream") {
  if (need <= cap) return LB2_OK;
  const cudaError_t e = regrow(p, cap, need, 16);
  if (e == cudaErrorMemoryAllocation) {
    cudaGetLastError();
    ctx->err = std::string(what) + " does not fit in device memory";
    return LB2_E_CAPACITY;
  }
  CK(e);
  return LB2_OK;
}

// LB2_INFLATE_SPAN_KB (default 128): the nominal span, read at each run
static bool ifl_span(lb2_ctx *ctx, uint64_t &span) {
  span = 128 << 10;
  if (const char *v = getenv("LB2_INFLATE_SPAN_KB")) {
    const long kb = atol(v);
    if (kb < 1) { ctx->err = "LB2_INFLATE_SPAN_KB must be a positive number of KB"; return false; }
    span = (uint64_t)kb << 10;
  }
  return true;
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
      (e = cudaMalloc(&d->d_crc, sizeof(uint32_t))) != cudaSuccess || (e = cudaMalloc(&d->d_err, sizeof(int32_t))) != cudaSuccess ||
      (e = cudaMalloc(&d->d_first, 2 * sizeof(uint32_t))) != cudaSuccess) {
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
  cudaFree(d->d_chunk_crc); cudaFree(d->d_crc); cudaFree(d->d_err); cudaFree(d->d_find); cudaFree(d->d_first);
  for (auto &e : d->ev) if (e) cudaEventDestroy(e);
  if (d->stream) cudaStreamDestroy(d->stream);
  delete d;
}

}  // extern "C"

// The table path: one exact-stop span per entry, decoded into the arena with its result; true when Table::accept takes
// the results (d_jobs then holds the laid-out spans).  A table that does not fit on the device is refused like one
// that does not chain.
static int ifl_table(lb2_inflate *d, uint64_t n, const lb2_inflate_span *spans, uint32_t n_spans, ifl::Table &t,
                     lb2_inflate_stats &st, bool &accepted) {
  lb2_ctx *ctx = d->ctx;
  cudaStream_t s = d->stream;
  accepted = false;
  static_assert(sizeof(lb2_inflate_span) == sizeof(ifl::TableEntry), "seek-table entries");
  if (!t.init(reinterpret_cast<const ifl::TableEntry *>(spans), n_spans, n)) return LB2_OK;
  const uint64_t total = t.out_total;
  const uint64_t cap_arena = d->cap_arena;
  // a refused table leaves no trace: not its error message, nor output buffers grown to what it claimed (up to
  // MAX_RATIO x the input), which the search then allocates for the stream's real size
  auto refuse = [&]() {
    ctx->err.clear();
    if (d->cap_arena > cap_arena) {
      cudaFree(d->d_arena); cudaFree(d->d_out); cudaFree(d->d_chunk_crc);
      d->d_arena = nullptr; d->d_out = nullptr; d->d_chunk_crc = nullptr;
      d->cap_arena = d->cap_out = d->cap_chunks = 0;
    }
    return LB2_OK;
  };
  if (ifl_grow(ctx, &d->d_jobs, d->cap_jobs, n_spans) || ifl_grow(ctx, &d->d_res, d->cap_res, n_spans) ||
      ifl_grow(ctx, &d->d_arena, d->cap_arena, total) || ifl_grow(ctx, &d->d_out, d->cap_out, total) ||
      ifl_grow(ctx, &d->d_chunk_crc, d->cap_chunks, (total + GZ_CHUNK - 1) / GZ_CHUNK + 1))
    return refuse();
  std::vector<ifl::SpanResult> res(n_spans);
  CK(cudaMemcpyAsync(d->d_jobs, t.job.data(), n_spans * sizeof(ifl::SpanJob), cudaMemcpyHostToDevice, s));
  CK(cudaEventRecord(d->ev[0], s));
  launch_inflate_table_decode(d->d_in, d->d_jobs, n_spans, d->d_arena, d->d_res, s);
  CK(cudaGetLastError());
  CK(cudaEventRecord(d->ev[1], s));
  CK(cudaMemcpyAsync(res.data(), d->d_res, n_spans * sizeof(ifl::SpanResult), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  st.decode_ms += ifl_elapsed(d);
  accepted = t.accept(res.data());
  return accepted ? LB2_OK : refuse();
}

// The search path: candidates, count rounds and chain, then the decode of the confirmed spans into the arena.
// *total is the stream's output; d_jobs holds the laid-out spans.
static int ifl_search(lb2_inflate *d, uint64_t n, lb2_inflate_stats &st, std::vector<ifl::SpanJob> &used, uint64_t *total) {
  lb2_ctx *ctx = d->ctx;
  cudaStream_t s = d->stream;
  uint64_t span;
  if (!ifl_span(ctx, span)) return LB2_E_ARG;
  const uint32_t n_spans = n > span ? (uint32_t)((n + span - 1) / span) : 1;
  int rc;
  if ((rc = ifl_grow(ctx, &d->d_cand, d->cap_cand, n_spans)) || (rc = ifl_grow(ctx, &d->d_jobs, d->cap_jobs, n_spans)) ||
      (rc = ifl_grow(ctx, &d->d_res, d->cap_res, n_spans)) || (rc = ifl_grow(ctx, &d->d_find, d->cap_find, n_spans)))
    return rc;
  std::vector<ifl::FindJob> find;  // the one stream's nominal spans k >= 1
  for (uint32_t k = 1; k < n_spans; k++) find.push_back(ifl::FindJob{0, n, k, 0});
  if (!find.empty()) CK(cudaMemcpyAsync(d->d_find, find.data(), find.size() * sizeof(ifl::FindJob), cudaMemcpyHostToDevice, s));
  // candidates
  std::vector<uint64_t> cand(n_spans, ifl::KEY_NONE);
  CK(cudaEventRecord(d->ev[0], s));
  launch_inflate_find(d->d_in, span, d->d_find, (uint32_t)find.size(), d->d_cand, s);
  CK(cudaGetLastError());
  CK(cudaEventRecord(d->ev[1], s));
  if (n_spans > 1) CK(cudaMemcpyAsync(cand.data() + 1, d->d_cand, (n_spans - 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
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
    launch_inflate_count(d->d_in, d->d_jobs, (uint32_t)jobs.size(), d->d_res, s);
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
    return LB2_E_DATA;
  }
  *total = c.layout();
  const uint32_t n_used = (uint32_t)c.job.size();
  st.in_bytes = c.in_bytes();
  // 2 bytes per output byte for the u16 arena, 1 for the final bytes
  if ((rc = ifl_grow(ctx, &d->d_arena, d->cap_arena, *total)) || (rc = ifl_grow(ctx, &d->d_out, d->cap_out, *total)) ||
      (rc = ifl_grow(ctx, &d->d_chunk_crc, d->cap_chunks, (*total + GZ_CHUNK - 1) / GZ_CHUNK + 1)))
    return rc;
  CK(cudaMemcpyAsync(d->d_jobs, c.job.data(), n_used * sizeof(ifl::SpanJob), cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(d->d_err, 0, sizeof(int32_t), s));
  CK(cudaEventRecord(d->ev[0], s));
  launch_inflate_decode(d->d_in, d->d_jobs, n_used, d->d_arena, d->d_err, s);
  CK(cudaGetLastError());
  CK(cudaEventRecord(d->ev[1], s));
  CK(cudaEventSynchronize(d->ev[1]));
  st.decode_ms += ifl_elapsed(d);
  used.swap(c.job);
  return LB2_OK;
}

// lb2_inflate_run (no table) and lb2_inflate_run_table: upload, the table path if there is a table, the search path
// if there is none or it was refused, then resolve and CRC-32.
static int ifl_run(lb2_inflate *d, const void *h_in, uint64_t n, const lb2_inflate_span *spans, uint32_t n_table_spans,
                   uint64_t *out_n, lb2_inflate_stats *stats, uint32_t *n_table, uint32_t *n_refused) {
  if (!d) return LB2_E_ARG;
  lb2_ctx *ctx = d->ctx;
  if ((!h_in && n) || !out_n || (!spans && n_table_spans)) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  d->have = false;
  *out_n = 0;
  if (n_table) *n_table = 0;
  if (n_refused) *n_refused = 0;
  lb2_inflate_stats st{};
  uint64_t span;
  if (!ifl_span(ctx, span)) return LB2_E_ARG;
  cudaStream_t s = d->stream;
  int rc;
  if ((rc = ifl_grow(ctx, &d->d_in, d->cap_in, n))) return rc;
  // upload
  CK(cudaEventRecord(d->ev[0], s));
  if (n) CK(cudaMemcpyAsync(d->d_in, h_in, n, cudaMemcpyHostToDevice, s));
  CK(cudaEventRecord(d->ev[1], s));
  CK(cudaEventSynchronize(d->ev[1]));
  st.h2d_ms = ifl_elapsed(d);
  bool accepted = false;
  ifl::Table t;
  if (n_table_spans) {
    if ((rc = ifl_table(d, n, spans, n_table_spans, t, st, accepted))) return rc;
    if (n_table) *n_table = accepted;
    if (n_refused) *n_refused = !accepted;
  }
  std::vector<ifl::SpanJob> used;
  uint64_t total = 0;
  if (accepted) {
    used.swap(t.job);
    total = t.out_total;
    st.in_bytes = t.in_total;
    CK(cudaMemsetAsync(d->d_err, 0, sizeof(int32_t), s));
  } else if ((rc = ifl_search(d, n, st, used, &total))) {
    if (stats) *stats = st;
    return rc;
  }
  const uint32_t n_used = (uint32_t)used.size();
  st.n_spans = n_used;
  st.out_bytes = total;
  // resolve, CRC-32
  CK(cudaEventRecord(d->ev[0], s));
  const uint32_t span_range[2] = {0, n_used};
  CK(cudaMemcpyAsync(d->d_first, span_range, sizeof span_range, cudaMemcpyHostToDevice, s));
  launch_inflate_resolve(d->d_arena, d->d_out, d->d_jobs, n_used, d->d_first, 1, d->d_err, s);
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

extern "C" {

int lb2_inflate_run(lb2_inflate *d, const void *h_in, uint64_t n, uint64_t *out_n, lb2_inflate_stats *stats) {
  return ifl_run(d, h_in, n, nullptr, 0, out_n, stats, nullptr, nullptr);
}

int lb2_inflate_run_table(lb2_inflate *d, const void *h_in, uint64_t n, const lb2_inflate_span *spans, uint32_t n_spans,
                          uint64_t *out_n, lb2_inflate_stats *stats, uint32_t *n_table, uint32_t *n_refused) {
  return ifl_run(d, h_in, n, spans, n_spans, out_n, stats, n_table, n_refused);
}

int lb2_inflate_device_output(lb2_inflate *d, const void **d_out, uint64_t *n) {
  if (!d) return LB2_E_ARG;
  lb2_ctx *ctx = d->ctx;
  if (!d_out || !n) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  if (!d->have) { ctx->err = "lb2_inflate_device_output: no decoded stream (lb2_inflate_run failed or was not called)"; return LB2_E_STATE; }
  *d_out = d->out_n ? d->d_out : nullptr;
  *n = d->out_n;
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

// ---------------------------------------------------------------------------- zip reader
// The inflate pipeline over a member table (ifl::Batch in inflate_core.cuh).  The archive bytes are uploaded once;
// STORED members are copied, one-span members decoded whole, larger ones run find / count rounds / decode / resolve
// with every member's spans in the same launches; then the writer's CRC and scan kernels give each member's CRC-32.
static_assert(sizeof(ifl::Member) == 40 && sizeof(lb2_unzip_member) == 32, "member table entries");

struct lb2_unzip {
  lb2_ctx *ctx = nullptr;
  cudaStream_t stream = nullptr;
  uint8_t *d_in = nullptr, *d_out = nullptr, *d_tab = nullptr;
  uint16_t *d_arena = nullptr;
  uint64_t *d_cand = nullptr, *d_chunk_off = nullptr;
  ifl::FindJob *d_find = nullptr;
  ifl::SpanJob *d_jobs = nullptr, *d_small = nullptr;
  ifl::SpanResult *d_res = nullptr;
  ifl::Member *d_members = nullptr;
  uint32_t *d_idx = nullptr, *d_first = nullptr, *d_chunk_crc = nullptr, *d_zero = nullptr;
  int32_t *d_status = nullptr;
  GzSegResult *d_seg = nullptr;
  GzResult *d_gres = nullptr;
  uint64_t cap_in = 0, cap_out = 0, cap_tab = 0, cap_arena = 0, cap_cand = 0, cap_chunk_off = 0, cap_find = 0, cap_jobs = 0,
           cap_small = 0, cap_res = 0, cap_members = 0, cap_idx = 0, cap_first = 0, cap_chunk_crc = 0, cap_zero = 0,
           cap_status = 0, cap_seg = 0, cap_gres = 0;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  uint64_t out_n = 0;
  bool have = false;
};

static float uz_elapsed(lb2_unzip *u) {
  float ms = 0;
  cudaEventElapsedTime(&ms, u->ev[0], u->ev[1]);
  return ms;
}

extern "C" {

int lb2_unzip_create(lb2_ctx *ctx, uint32_t flags, lb2_unzip **out) {
  if (!ctx || !out) { if (ctx) ctx->err = "NULL argument"; return LB2_E_ARG; }
  *out = nullptr;
  if (flags) { ctx->err = "lb2_unzip_create: no flags are defined"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  lb2_unzip *u = new lb2_unzip();
  u->ctx = ctx;
  cudaError_t e;
  if ((e = cudaStreamCreateWithFlags(&u->stream, cudaStreamNonBlocking)) != cudaSuccess ||
      (e = cudaEventCreate(&u->ev[0])) != cudaSuccess || (e = cudaEventCreate(&u->ev[1])) != cudaSuccess) {
    ctx->err = std::string("lb2_unzip_create: ") + cudaGetErrorString(e);
    lb2_unzip_destroy(u);
    return LB2_E_CUDA;
  }
  *out = u;
  return LB2_OK;
}

void lb2_unzip_destroy(lb2_unzip *u) {
  if (!u) return;
  cudaSetDevice(u->ctx->device);
  if (u->stream) cudaStreamSynchronize(u->stream);
  cudaFree(u->d_in); cudaFree(u->d_out); cudaFree(u->d_tab); cudaFree(u->d_arena); cudaFree(u->d_cand);
  cudaFree(u->d_chunk_off); cudaFree(u->d_find); cudaFree(u->d_jobs); cudaFree(u->d_small); cudaFree(u->d_res);
  cudaFree(u->d_members); cudaFree(u->d_idx); cudaFree(u->d_first); cudaFree(u->d_chunk_crc); cudaFree(u->d_zero);
  cudaFree(u->d_status); cudaFree(u->d_seg); cudaFree(u->d_gres);
  for (auto &e : u->ev) if (e) cudaEventDestroy(e);
  if (u->stream) cudaStreamDestroy(u->stream);
  delete u;
}

}  // extern "C"

// lb2_unzip_run (no tables) and lb2_unzip_run_table: members with an accepted seek table are decoded from it and
// resolved with the search path's spans; every other member (a refused table's included) takes the path it takes
// without one.
static int uz_run(lb2_unzip *u, const void *h_in, uint64_t n, const lb2_unzip_member *members, uint32_t n_members,
                  const uint32_t *span_first, const lb2_inflate_span *spans, uint64_t *out_n, lb2_unzip_result *results,
                  lb2_unzip_stats *stats, uint32_t *n_table, uint32_t *n_refused) {
  if (!u) return LB2_E_ARG;
  lb2_ctx *ctx = u->ctx;
  if ((!h_in && n) || !out_n || (n_members && (!members || !results)) || (span_first && !spans && span_first[n_members])) {
    ctx->err = "NULL argument";
    return LB2_E_ARG;
  }
  if (n_table) *n_table = 0;
  if (n_refused) *n_refused = 0;
  u->have = false;
  *out_n = 0;
  // everything the archive says is checked before any launch
  std::vector<ifl::Member> m(n_members);
  uint64_t total = 0, n_chunks = 0;
  for (uint32_t i = 0; i < n_members; i++) {
    const lb2_unzip_member &x = members[i];
    const std::string which = "lb2_unzip_run: member " + std::to_string(i);
    if (x.method != 0 && x.method != 8) { ctx->err = which + ": method " + std::to_string(x.method) + " is not 0 or 8"; return LB2_E_ARG; }
    if (x.body_off > n || x.body_len > n - x.body_off) { ctx->err = which + ": body outside the buffer"; return LB2_E_ARG; }
    if (x.size > UINT64_MAX - 32 - total) { ctx->err = which + ": output size overflows"; return LB2_E_ARG; }
    m[i] = ifl::Member{x.body_off, x.body_len, total, x.size, x.crc32, x.method};
    total = (total + x.size + 15) & ~15ull;  // 16-byte-aligned output offsets (the CRC kernel's vector loads)
    n_chunks += x.size ? (x.size + GZ_CHUNK - 1) / GZ_CHUNK : 1;
  }
  if (n_chunks > UINT32_MAX / 2) { ctx->err = "lb2_unzip_run: too many output chunks"; return LB2_E_ARG; }
  uint64_t span;
  if (!ifl_span(ctx, span)) return LB2_E_ARG;
  CK(cudaSetDevice(ctx->device));
  lb2_unzip_stats st{};
  st.n_members = n_members;
  st.in_bytes = n;
  // seek tables, checked on the host: a DEFLATE member that would take the search pipeline (more than one span) and
  // whose entries add up to its body and recorded size.  A one-span member is decoded whole by one thread anyway.
  std::vector<uint8_t> tabled(n_members, 0);
  std::vector<ifl::Table> tables;
  std::vector<uint32_t> table_member;
  uint32_t refused = 0;
  for (uint32_t i = 0; span_first && i < n_members; i++) {
    const uint32_t k = span_first[i + 1] - span_first[i];
    const ifl::Member &x = m[i];
    if (!k || (x.method == 8 && x.in_len <= span)) continue;
    ifl::Table t;
    if (span_first[i + 1] < span_first[i] || x.method != 8 ||
        !t.init(reinterpret_cast<const ifl::TableEntry *>(spans + span_first[i]), k, x.in_len, x.in_off, x.out_off, i) ||
        t.in_total != x.in_len || t.out_total != x.out_len) {
      refused++;
      continue;
    }
    tables.push_back(std::move(t));
    table_member.push_back(i);
  }
  ifl::Batch b;  // sized here for every member; set up again below without those a table decodes
  b.init(m.data(), n_members, span);
  st.n_stored = (uint32_t)b.stored.size();
  st.n_small = (uint32_t)b.small.size();
  st.n_large = (uint32_t)b.large.size();
  const char *what = "lb2_unzip_run: the archive";
  const uint64_t tab = n_chunks * sizeof(GzChunk) + (uint64_t)n_members * sizeof(GzSeg);
  int rc;
  if ((rc = ifl_grow(ctx, &u->d_in, u->cap_in, n, what)) || (rc = ifl_grow(ctx, &u->d_out, u->cap_out, total, what)) ||
      (rc = ifl_grow(ctx, &u->d_members, u->cap_members, n_members, what)) ||
      (rc = ifl_grow(ctx, &u->d_status, u->cap_status, n_members, what)) ||
      (rc = ifl_grow(ctx, &u->d_idx, u->cap_idx, b.stored.size(), what)) ||
      (rc = ifl_grow(ctx, &u->d_small, u->cap_small, b.small.size(), what)) ||
      (rc = ifl_grow(ctx, &u->d_find, u->cap_find, b.find.size(), what)) ||
      (rc = ifl_grow(ctx, &u->d_cand, u->cap_cand, b.find.size(), what)) ||
      (rc = ifl_grow(ctx, &u->d_tab, u->cap_tab, tab, what)) ||
      (rc = ifl_grow(ctx, &u->d_chunk_crc, u->cap_chunk_crc, n_chunks, what)) ||
      (rc = ifl_grow(ctx, &u->d_zero, u->cap_zero, 2 * n_chunks + 1, what)) ||
      (rc = ifl_grow(ctx, &u->d_chunk_off, u->cap_chunk_off, n_chunks, what)) ||
      (rc = ifl_grow(ctx, &u->d_seg, u->cap_seg, n_members, what)) || (rc = ifl_grow(ctx, &u->d_gres, u->cap_gres, 1, what)))
    return rc;
  cudaStream_t s = u->stream;
  // upload: the archive, the member table and the host-known statuses
  CK(cudaEventRecord(u->ev[0], s));
  if (n) CK(cudaMemcpyAsync(u->d_in, h_in, n, cudaMemcpyHostToDevice, s));
  CK(cudaEventRecord(u->ev[1], s));
  if (n_members) {
    CK(cudaMemcpyAsync(u->d_members, m.data(), n_members * sizeof(ifl::Member), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(u->d_status, b.status.data(), n_members * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  }
  CK(cudaStreamSynchronize(s));
  st.h2d_ms = uz_elapsed(u);
  // the seek-table members: one exact-stop span per entry into the arena, then Table::accept per member
  std::vector<ifl::SpanJob> table_jobs;
  std::vector<uint32_t> table_first{0};
  if (!tables.empty()) {
    std::vector<ifl::SpanJob> all;
    for (const ifl::Table &t : tables) all.insert(all.end(), t.job.begin(), t.job.end());
    if ((rc = ifl_grow(ctx, &u->d_arena, u->cap_arena, total, what)) || (rc = ifl_grow(ctx, &u->d_jobs, u->cap_jobs, all.size(), what)) ||
        (rc = ifl_grow(ctx, &u->d_res, u->cap_res, all.size(), what)))
      return rc;
    std::vector<ifl::SpanResult> res(all.size());
    CK(cudaMemcpyAsync(u->d_jobs, all.data(), all.size() * sizeof(ifl::SpanJob), cudaMemcpyHostToDevice, s));
    CK(cudaEventRecord(u->ev[0], s));
    launch_inflate_table_decode(u->d_in, u->d_jobs, (uint32_t)all.size(), u->d_arena, u->d_res, s);
    CK(cudaGetLastError());
    CK(cudaEventRecord(u->ev[1], s));
    CK(cudaMemcpyAsync(res.data(), u->d_res, res.size() * sizeof(ifl::SpanResult), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    st.decode_ms += uz_elapsed(u);
    size_t at = 0;
    for (size_t i = 0; i < tables.size(); i++) {
      if (tables[i].accept(res.data() + at)) {
        tabled[table_member[i]] = 1;
        table_jobs.insert(table_jobs.end(), tables[i].job.begin(), tables[i].job.end());
        table_first.push_back((uint32_t)table_jobs.size());
      } else {
        refused++;
      }
      at += tables[i].job.size();
    }
  }
  if (n_table) *n_table = (uint32_t)table_first.size() - 1;
  if (n_refused) *n_refused = refused;
  if (table_first.size() > 1) {  // the accepted members leave every other path (the buffers above are large enough)
    b.init(m.data(), n_members, span, tabled.data());
    st.n_small = (uint32_t)b.small.size();
    st.n_large = (uint32_t)b.large.size();
  }
  if (!b.stored.empty()) CK(cudaMemcpyAsync(u->d_idx, b.stored.data(), b.stored.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
  if (!b.small.empty()) CK(cudaMemcpyAsync(u->d_small, b.small.data(), b.small.size() * sizeof(ifl::SpanJob), cudaMemcpyHostToDevice, s));
  if (!b.find.empty()) CK(cudaMemcpyAsync(u->d_find, b.find.data(), b.find.size() * sizeof(ifl::FindJob), cudaMemcpyHostToDevice, s));
  // STORED members, then the one-span members
  CK(cudaEventRecord(u->ev[0], s));
  launch_unzip_copy(u->d_in, u->d_members, u->d_idx, (uint32_t)b.stored.size(), u->d_out, s);
  CK(cudaGetLastError());
  CK(cudaEventRecord(u->ev[1], s));
  CK(cudaEventSynchronize(u->ev[1]));
  st.copy_ms = uz_elapsed(u);
  CK(cudaEventRecord(u->ev[0], s));
  launch_unzip_small(u->d_in, u->d_small, (uint32_t)b.small.size(), u->d_out, u->d_status, s);
  CK(cudaGetLastError());
  CK(cudaEventRecord(u->ev[1], s));
  CK(cudaEventSynchronize(u->ev[1]));
  st.small_ms = uz_elapsed(u);
  // larger members: candidates, then count rounds with one chain per member
  std::vector<ifl::SpanJob> jobs;
  std::vector<uint32_t> first{0};
  if (!b.large.empty()) {
    std::vector<uint64_t> cand(b.find.size());
    CK(cudaEventRecord(u->ev[0], s));
    launch_inflate_find(u->d_in, span, u->d_find, (uint32_t)b.find.size(), u->d_cand, s);
    CK(cudaGetLastError());
    CK(cudaEventRecord(u->ev[1], s));
    if (!cand.empty()) CK(cudaMemcpyAsync(cand.data(), u->d_cand, cand.size() * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    st.find_ms = uz_elapsed(u);
    b.start_chains(cand.data(), span);
    std::vector<ifl::SpanResult> res;
    std::vector<std::pair<uint32_t, uint32_t>> ref;
    while (b.pending(jobs, ref)) {
      if ((rc = ifl_grow(ctx, &u->d_jobs, u->cap_jobs, jobs.size(), what)) || (rc = ifl_grow(ctx, &u->d_res, u->cap_res, jobs.size(), what)))
        return rc;
      res.resize(jobs.size());
      CK(cudaMemcpyAsync(u->d_jobs, jobs.data(), jobs.size() * sizeof(ifl::SpanJob), cudaMemcpyHostToDevice, s));
      CK(cudaEventRecord(u->ev[0], s));
      launch_inflate_count(u->d_in, u->d_jobs, (uint32_t)jobs.size(), u->d_res, s);
      CK(cudaGetLastError());
      CK(cudaEventRecord(u->ev[1], s));
      CK(cudaMemcpyAsync(res.data(), u->d_res, res.size() * sizeof(ifl::SpanResult), cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      st.count_ms += uz_elapsed(u);
      b.set_results(ref, res.data());
    }
    st.n_rounds = b.n_rounds;
    st.n_rejected = b.n_rejected();
    st.n_absorbed = b.n_absorbed();
    // the members whose chains ended at their recorded sizes
    b.layout(jobs, first);
  }
  // decode the search path's spans into the u16 arena at their output offsets, then resolve them with the accepted
  // seek-table members' spans (decoded above)
  const uint32_t n_search = (uint32_t)jobs.size();
  for (size_t i = 1; i < table_first.size(); i++) first.push_back(n_search + table_first[i]);
  jobs.insert(jobs.end(), table_jobs.begin(), table_jobs.end());
  st.n_spans = (uint32_t)jobs.size();
  const uint32_t n_dec = (uint32_t)first.size() - 1;
  if (n_dec) {
    if ((rc = ifl_grow(ctx, &u->d_arena, u->cap_arena, total, what)) || (rc = ifl_grow(ctx, &u->d_jobs, u->cap_jobs, jobs.size(), what)) ||
        (rc = ifl_grow(ctx, &u->d_first, u->cap_first, first.size(), what)))
      return rc;
    CK(cudaMemcpyAsync(u->d_jobs, jobs.data(), jobs.size() * sizeof(ifl::SpanJob), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(u->d_first, first.data(), first.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CK(cudaEventRecord(u->ev[0], s));
    launch_inflate_decode(u->d_in, u->d_jobs, n_search, u->d_arena, u->d_status, s);
    CK(cudaGetLastError());
    CK(cudaEventRecord(u->ev[1], s));
    CK(cudaEventSynchronize(u->ev[1]));
    st.decode_ms += uz_elapsed(u);
    CK(cudaEventRecord(u->ev[0], s));
    launch_inflate_resolve(u->d_arena, u->d_out, u->d_jobs, (uint32_t)jobs.size(), u->d_first, n_dec, u->d_status, s);
    CK(cudaGetLastError());
    CK(cudaEventRecord(u->ev[1], s));
    CK(cudaEventSynchronize(u->ev[1]));
    st.resolve_ms = uz_elapsed(u);
  }
  // CRC-32 of every member: the writer's chunk table over the output, one segment per member
  std::vector<GzSegResult> seg(n_members);
  std::vector<int32_t> dev_status(n_members);
  if (n_members) {
    std::vector<uint8_t> h_tab(tab);
    GzChunk *chunks = reinterpret_cast<GzChunk *>(h_tab.data());
    GzSeg *segs = reinterpret_cast<GzSeg *>(h_tab.data() + n_chunks * sizeof(GzChunk));
    uint32_t c = 0;
    for (uint32_t i = 0; i < n_members; i++) {
      segs[i] = GzSeg{m[i].out_off, m[i].out_len, c, GZ_SEG_ENDS};
      uint64_t p = 0;
      do {
        const uint32_t len = (uint32_t)std::min<uint64_t>(GZ_CHUNK, m[i].out_len - p);
        chunks[c++] = GzChunk{m[i].out_off + p, len, 0, i, 0};
        p += len;
      } while (p < m[i].out_len);
    }
    GzPieceArgs a{};
    a.in = u->d_out; a.n = total; a.n_chunks = c; a.n_segs = n_members;
    a.chunks = reinterpret_cast<const GzChunk *>(u->d_tab);
    a.segs = reinterpret_cast<const GzSeg *>(u->d_tab + n_chunks * sizeof(GzChunk));
    a.chunk_size = u->d_zero; a.chunk_mode = u->d_zero + n_chunks; a.crc_state = u->d_zero + 2 * n_chunks;
    a.chunk_crc = u->d_chunk_crc; a.chunk_off = u->d_chunk_off; a.seg_res = u->d_seg; a.res = u->d_gres;
    CK(cudaMemcpyAsync(u->d_tab, h_tab.data(), tab, cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(u->d_zero, 0, (2 * n_chunks + 1) * sizeof(uint32_t), s));
    CK(cudaEventRecord(u->ev[0], s));
    launch_segment_crc32(a, s);
    CK(cudaGetLastError());
    CK(cudaEventRecord(u->ev[1], s));
    CK(cudaMemcpyAsync(seg.data(), u->d_seg, n_members * sizeof(GzSegResult), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(dev_status.data(), u->d_status, n_members * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    st.crc_ms = uz_elapsed(u);
  }
  for (uint32_t i = 0; i < n_members; i++) {
    // a status found on the host stands; a device one is the small kernel's, or a large member's span status (< 0)
    int32_t r = b.status[i] != ifl::MS_OK ? b.status[i] : dev_status[i] < 0 ? (int32_t)ifl::MS_BAD_DATA : dev_status[i];
    if (r == ifl::MS_OK && seg[i].crc32 != m[i].crc32) r = ifl::MS_BAD_CRC;
    results[i].out_off = m[i].out_off;
    results[i].crc32 = seg[i].crc32;
    results[i].status = r;
    st.n_bad += r != ifl::MS_OK;
    st.out_bytes += m[i].out_len;
  }
  if (stats) *stats = st;
  u->out_n = total;
  u->have = true;
  *out_n = total;
  return LB2_OK;
}

extern "C" {

int lb2_unzip_run(lb2_unzip *u, const void *h_in, uint64_t n, const lb2_unzip_member *members, uint32_t n_members,
                  uint64_t *out_n, lb2_unzip_result *results, lb2_unzip_stats *stats) {
  return uz_run(u, h_in, n, members, n_members, nullptr, nullptr, out_n, results, stats, nullptr, nullptr);
}

int lb2_unzip_run_table(lb2_unzip *u, const void *h_in, uint64_t n, const lb2_unzip_member *members, uint32_t n_members,
                        const uint32_t *span_first, const lb2_inflate_span *spans, uint64_t *out_n,
                        lb2_unzip_result *results, lb2_unzip_stats *stats, uint32_t *n_table, uint32_t *n_refused) {
  if (u && !span_first) { u->ctx->err = "NULL argument"; return LB2_E_ARG; }
  return uz_run(u, h_in, n, members, n_members, span_first, spans, out_n, results, stats, n_table, n_refused);
}

int lb2_unzip_device_output(lb2_unzip *u, const void **d_out, uint64_t *n) {
  if (!u) return LB2_E_ARG;
  lb2_ctx *ctx = u->ctx;
  if (!d_out || !n) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  if (!u->have) { ctx->err = "lb2_unzip_device_output: no decoded batch (lb2_unzip_run failed or was not called)"; return LB2_E_STATE; }
  *d_out = u->d_out;
  *n = u->out_n;
  return LB2_OK;
}

int lb2_unzip_read(lb2_unzip *u, void *h_out, uint64_t cap) {
  if (!u) return LB2_E_ARG;
  lb2_ctx *ctx = u->ctx;
  if (!u->have) { ctx->err = "lb2_unzip_read: no decoded batch (lb2_unzip_run failed or was not called)"; return LB2_E_STATE; }
  if (cap < u->out_n) { ctx->err = "lb2_unzip_read: buffer smaller than the decoded batch"; return LB2_E_CAPACITY; }
  if (!h_out && u->out_n) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  if (u->out_n) CK(cudaMemcpy(h_out, u->d_out, u->out_n, cudaMemcpyDeviceToHost));
  return LB2_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------- tar index
// The walk kernel (tar.cu) on the context's stream; ranges and bytes land in one scratch allocation of the call.
#include "tar_walk.cuh"
static_assert(sizeof(lb2_tar_range) == sizeof(tarw::Range), "the walk kernel writes lb2_tar_range records");

extern "C" {

int lb2_tar_index(lb2_ctx *ctx, const void *d_tar, uint64_t n, lb2_tar_range *ranges, uint32_t max_ranges, uint32_t *n_ranges,
                  void *h_bytes, uint64_t bytes_cap, uint64_t *n_bytes, lb2_tar_index_stats *stats) {
  if (!ctx) return LB2_E_ARG;
  if ((!d_tar && n) || !n_ranges || !n_bytes || (!ranges && max_ranges) || (!h_bytes && bytes_cap)) {
    ctx->err = "NULL argument";
    return LB2_E_ARG;
  }
  if (reinterpret_cast<uintptr_t>(d_tar) & 15) { ctx->err = "lb2_tar_index: d_tar must be 16-byte aligned"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  const uint64_t r_bytes = (uint64_t)max_ranges * sizeof(lb2_tar_range);
  uint8_t *d_ws = nullptr;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  TarWalkOut out{};
  float ms = 0;
  cudaError_t e = cudaMalloc(&d_ws, sizeof(TarWalkOut) + r_bytes + bytes_cap);
  if (e == cudaSuccess) e = cudaEventCreate(&ev[0]);
  if (e == cudaSuccess) e = cudaEventCreate(&ev[1]);
  if (e == cudaSuccess) e = cudaEventRecord(ev[0], ctx->stream);
  if (e == cudaSuccess) {
    launch_tar_walk(static_cast<const uint8_t *>(d_tar), n, d_ws + sizeof(TarWalkOut), max_ranges,
                    d_ws + sizeof(TarWalkOut) + r_bytes, bytes_cap, reinterpret_cast<TarWalkOut *>(d_ws), ctx->stream);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaEventRecord(ev[1], ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&out, d_ws, sizeof out, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, ev[0], ev[1]);
  const bool fits = out.n_ranges <= max_ranges && out.n_bytes <= bytes_cap;
  if (e == cudaSuccess && fits && out.n_ranges)
    e = cudaMemcpy(ranges, d_ws + sizeof(TarWalkOut), out.n_ranges * sizeof(lb2_tar_range), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && fits && out.n_bytes)
    e = cudaMemcpy(h_bytes, d_ws + sizeof(TarWalkOut) + r_bytes, out.n_bytes, cudaMemcpyDeviceToHost);
  cudaFree(d_ws);
  for (auto &v : ev) if (v) cudaEventDestroy(v);
  if (e != cudaSuccess) { ctx->err = std::string("lb2_tar_index: ") + cudaGetErrorString(e); return LB2_E_CUDA; }
  *n_ranges = out.n_ranges > UINT32_MAX ? UINT32_MAX : (uint32_t)out.n_ranges;
  *n_bytes = out.n_bytes;
  if (stats) *stats = lb2_tar_index_stats{out.members, out.stop_off, out.reason, ms};
  if (!fits) { ctx->err = "lb2_tar_index: ranges or bytes exceed the capacity given (*n_ranges, *n_bytes needed)"; return LB2_E_CAPACITY; }
  return LB2_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------- dynamic sections
// The count and write kernels (elf_deps.cu) on the context's stream, the exclusive scan of the counts on the host in
// between; everything lives in one scratch allocation of the call.
#include "elf_deps.cuh"
static_assert(sizeof(lb2_elf_object) == sizeof(elfd::Object), "the count kernel writes lb2_elf_object records");
static_assert(sizeof(lb2_elf_record) == sizeof(elfd::Record), "the write kernel writes lb2_elf_record records");

extern "C" {

int lb2_elf_deps(lb2_ctx *ctx, const uint64_t *d_ptrs, const uint64_t *sizes, uint32_t n, lb2_elf_object *objects,
                 lb2_elf_record *records, uint32_t max_records, uint32_t *n_records, void *h_pool, uint64_t pool_cap,
                 uint64_t *pool_bytes, lb2_elf_deps_stats *stats) {
  if (!ctx) return LB2_E_ARG;
  if ((n && (!d_ptrs || !sizes || !objects)) || !n_records || !pool_bytes || (!records && max_records) || (!h_pool && pool_cap)) {
    ctx->err = "NULL argument";
    return LB2_E_ARG;
  }
  for (uint32_t i = 0; i < n; i++)
    if (!d_ptrs[i] && sizes[i]) { ctx->err = "lb2_elf_deps: a NULL object address"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  const uint64_t job_bytes = 2 * sizeof(uint64_t) * (uint64_t)n, obj_bytes = sizeof(lb2_elf_object) * (uint64_t)n;
  const uint64_t rec_bytes = sizeof(lb2_elf_record) * (uint64_t)max_records, head = job_bytes + obj_bytes;
  uint8_t *d_ws = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  float ms[2] = {0, 0};
  uint64_t total_rec = 0, total_pool = 0, down = 0;
  bool fits = true;
  cudaError_t e = cudaMalloc(&d_ws, head + rec_bytes + pool_cap + 16);
  for (auto &v : ev)
    if (e == cudaSuccess) e = cudaEventCreate(&v);
  const uint64_t *d_p = reinterpret_cast<const uint64_t *>(d_ws), *d_s = d_p + n;
  void *d_obj = d_ws + job_bytes;
  if (e == cudaSuccess && n) e = cudaMemcpyAsync(d_ws, d_ptrs, job_bytes / 2, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess && n) e = cudaMemcpyAsync(d_ws + job_bytes / 2, sizes, job_bytes / 2, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaEventRecord(ev[0], ctx->stream);
  if (e == cudaSuccess) {
    launch_elf_deps_count(d_p, d_s, n, d_obj, ctx->stream);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaEventRecord(ev[1], ctx->stream);
  if (e == cudaSuccess && n) e = cudaMemcpyAsync(objects, d_obj, obj_bytes, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (e == cudaSuccess) e = cudaEventElapsedTime(&ms[0], ev[0], ev[1]);
  if (e == cudaSuccess) {
    down += obj_bytes;
    for (uint32_t i = 0; i < n; i++) {  // the exclusive scan
      objects[i].first_record = (uint32_t)total_rec;
      objects[i].pool_off = total_pool;
      total_rec += objects[i].n_records;
      total_pool += objects[i].pool_len;
    }
    fits = total_rec <= max_records && total_pool <= pool_cap;
    if (total_rec > UINT32_MAX) fits = false;
  }
  if (e == cudaSuccess && fits && total_rec) {
    e = cudaMemcpyAsync(d_obj, objects, obj_bytes, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaEventRecord(ev[2], ctx->stream);
    if (e == cudaSuccess) {
      launch_elf_deps_write(d_p, d_s, n, d_obj, d_ws + head, d_ws + head + rec_bytes, pool_cap, ctx->stream);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaEventRecord(ev[3], ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(records, d_ws + head, total_rec * sizeof(lb2_elf_record), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess && total_pool) e = cudaMemcpyAsync(h_pool, d_ws + head + rec_bytes, total_pool, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms[1], ev[2], ev[3]);
    down += total_rec * sizeof(lb2_elf_record) + total_pool;
  }
  cudaFree(d_ws);
  for (auto &v : ev) if (v) cudaEventDestroy(v);
  if (e != cudaSuccess) { ctx->err = std::string("lb2_elf_deps: ") + cudaGetErrorString(e); return LB2_E_CUDA; }
  *n_records = total_rec > UINT32_MAX ? UINT32_MAX : (uint32_t)total_rec;
  *pool_bytes = total_pool;
  if (stats) *stats = lb2_elf_deps_stats{total_rec, total_pool, down, ms[0] + ms[1]};
  if (!fits) { ctx->err = "lb2_elf_deps: records or pool exceed the capacity given (*n_records, *pool_bytes needed)"; return LB2_E_CAPACITY; }
  return LB2_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------- symbol lookups
// The index, reference and resolve kernels (elf_syms.cu) on the context's stream.  The arena is a list of device
// chunks; an index call takes one block for the tables of its batch and one for their references, each object's
// pieces at 8-byte alignment.  Scratch of a call lives in one allocation freed before it returns.
#include "elf_syms.cuh"
static_assert(sizeof(lb2_sym_object) == sizeof(elfs::Object), "the index kernels write lb2_sym_object records");
static_assert(sizeof(lb2_sym_job) == sizeof(elfs::Job) && sizeof(lb2_sym_miss) == sizeof(elfs::Miss), "resolve records");
static_assert(sizeof(lb2_sym_query) == sizeof(elfs::Query) && sizeof(lb2_sym_found) == sizeof(elfs::Found) &&
              LB2_SYM_NOT_FOUND == elfs::NOT_FOUND, "find records");

struct lb2_syms {
  lb2_ctx *ctx = nullptr;
  std::vector<void *> chunks;
  uint8_t *cur = nullptr;
  uint64_t used = 0, cap = 0, total = 0;
  std::vector<lb2_sym_object> objs;
};

namespace {
constexpr uint64_t SYM_CHUNK = 64ull << 20;

// n bytes of the arena (8-aligned), or nullptr when the device has no room for a new chunk
uint8_t *syms_alloc(lb2_syms *s, uint64_t n) {
  n = (n + 255) & ~255ull;
  if (!n) return nullptr;
  if (s->used + n > s->cap) {
    const uint64_t c = n > SYM_CHUNK ? n : SYM_CHUNK;
    void *p = nullptr;
    if (cudaMalloc(&p, c) != cudaSuccess) {
      cudaGetLastError();
      return nullptr;
    }
    s->chunks.push_back(p);
    s->cur = static_cast<uint8_t *>(p);
    s->used = 0;
    s->cap = c;
    s->total += c;
  }
  uint8_t *p = s->cur + s->used;
  s->used += n;
  return p;
}

struct SymScratch {  // one device allocation and the events of a call
  uint8_t *d = nullptr;
  cudaEvent_t ev[8] = {};
  cudaError_t e = cudaSuccess;
  explicit SymScratch(uint64_t bytes) {
    e = cudaMalloc(&d, bytes ? bytes : 16);
    for (auto &v : ev)
      if (e == cudaSuccess) e = cudaEventCreate(&v);
  }
  float ms(int a, int b) {
    float t = 0;
    if (e == cudaSuccess) e = cudaEventElapsedTime(&t, ev[a], ev[b]);
    return t;
  }
  ~SymScratch() {
    cudaFree(d);
    for (auto &v : ev) if (v) cudaEventDestroy(v);
  }
};
}  // namespace

extern "C" {

int lb2_syms_create(lb2_ctx *ctx, lb2_syms **out) {
  if (!ctx) return LB2_E_ARG;
  if (!out) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  *out = new lb2_syms;
  (*out)->ctx = ctx;
  return LB2_OK;
}

void lb2_syms_destroy(lb2_syms *s) {
  if (!s) return;
  cudaSetDevice(s->ctx->device);
  for (void *p : s->chunks) cudaFree(p);
  delete s;
}

int lb2_syms_index(lb2_syms *s, const uint64_t *d_ptrs, const uint64_t *sizes, uint32_t n, uint32_t *ids,
                   lb2_sym_object *objects, lb2_syms_stats *stats) {
  if (!s) return LB2_E_ARG;
  lb2_ctx *ctx = s->ctx;
  if (n && (!d_ptrs || !sizes || !ids || !objects)) { ctx->err = "NULL argument"; return LB2_E_ARG; }
  for (uint32_t i = 0; i < n; i++)
    if (!d_ptrs[i] && sizes[i]) { ctx->err = "lb2_syms_index: a NULL object address"; return LB2_E_ARG; }
  lb2_syms_stats st{};
  if (!n) { if (stats) *stats = st; return LB2_OK; }
  CK(cudaSetDevice(ctx->device));
  const uint64_t job_bytes = 2 * sizeof(uint64_t) * (uint64_t)n, obj_bytes = sizeof(lb2_sym_object) * (uint64_t)n;
  SymScratch w(job_bytes + obj_bytes + 8 * ((uint64_t)n + 1));
  cudaError_t &e = w.e;
  const uint64_t *d_p = reinterpret_cast<const uint64_t *>(w.d), *d_s = d_p + n;
  void *d_obj = w.d + job_bytes;
  uint64_t *d_base = reinterpret_cast<uint64_t *>(w.d + job_bytes + obj_bytes);
  cudaStream_t q = ctx->stream;
  if (e == cudaSuccess) e = cudaMemcpyAsync(w.d, d_ptrs, job_bytes / 2, cudaMemcpyHostToDevice, q);
  if (e == cudaSuccess) e = cudaMemcpyAsync(w.d + job_bytes / 2, sizes, job_bytes / 2, cudaMemcpyHostToDevice, q);
  if (e == cudaSuccess) e = cudaEventRecord(w.ev[0], q);
  if (e == cudaSuccess) { launch_syms_index_count(d_p, d_s, n, d_obj, q); e = cudaGetLastError(); }
  if (e == cudaSuccess) e = cudaEventRecord(w.ev[1], q);
  if (e == cudaSuccess) e = cudaMemcpyAsync(objects, d_obj, obj_bytes, cudaMemcpyDeviceToHost, q);
  if (e == cudaSuccess) e = cudaStreamSynchronize(q);
  st.bytes_up += job_bytes;
  st.bytes_down += obj_bytes;
  // the tables' block, and the relocation entries' prefix
  std::vector<uint64_t> base(n + 1, 0);
  uint64_t need = 0;
  for (uint32_t i = 0; i < n; i++) {
    base[i + 1] = base[i] + (objects[i].status == elfs::ST_OK ? objects[i].rela_n + objects[i].plt_n : 0);
    if (objects[i].status == elfs::ST_OK) need += elfs::tables(reinterpret_cast<const elfs::Object &>(objects[i])).end;
  }
  uint8_t *block = nullptr;
  if (e == cudaSuccess && need) {
    block = syms_alloc(s, need);
    if (!block) { ctx->err = "lb2_syms_index: no device memory for the symbol arena"; return LB2_E_CAPACITY; }
    uint64_t at = 0;
    for (uint32_t i = 0; i < n; i++)
      if (objects[i].status == elfs::ST_OK) {
        objects[i].arena = reinterpret_cast<uint64_t>(block + at);
        at += elfs::tables(reinterpret_cast<const elfs::Object &>(objects[i])).end;
      }
    e = cudaMemsetAsync(block, 0, need, q);
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_obj, objects, obj_bytes, cudaMemcpyHostToDevice, q);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_base, base.data(), 8 * ((uint64_t)n + 1), cudaMemcpyHostToDevice, q);
  st.bytes_up += obj_bytes + 8 * ((uint64_t)n + 1);
  if (e == cudaSuccess) e = cudaEventRecord(w.ev[2], q);
  if (e == cudaSuccess) { launch_syms_index_write(d_p, d_s, n, d_obj, q); e = cudaGetLastError(); }
  if (e == cudaSuccess) e = cudaEventRecord(w.ev[3], q);
  if (e == cudaSuccess) { launch_syms_refs(d_p, d_base, base[n], n, d_obj, q); e = cudaGetLastError(); }
  if (e == cudaSuccess) e = cudaEventRecord(w.ev[4], q);
  if (e == cudaSuccess) e = cudaMemcpyAsync(objects, d_obj, obj_bytes, cudaMemcpyDeviceToHost, q);
  if (e == cudaSuccess) e = cudaStreamSynchronize(q);
  st.bytes_down += obj_bytes;
  uint64_t nrefs = 0;
  for (uint32_t i = 0; i < n; i++) nrefs += objects[i].nrefs;
  if (e == cudaSuccess && nrefs) {
    uint8_t *refs = syms_alloc(s, nrefs * sizeof(elfs::Ref));
    if (!refs) { ctx->err = "lb2_syms_index: no device memory for the symbol arena"; return LB2_E_CAPACITY; }
    uint64_t at = 0;
    for (uint32_t i = 0; i < n; i++) {
      objects[i].refs = objects[i].nrefs ? reinterpret_cast<uint64_t>(refs + at) : 0;
      at += objects[i].nrefs * sizeof(elfs::Ref);
    }
    e = cudaMemcpyAsync(d_obj, objects, obj_bytes, cudaMemcpyHostToDevice, q);
    st.bytes_up += obj_bytes;
    if (e == cudaSuccess) e = cudaEventRecord(w.ev[5], q);
    if (e == cudaSuccess) { launch_syms_refs_write(n, d_obj, q); e = cudaGetLastError(); }
    if (e == cudaSuccess) e = cudaEventRecord(w.ev[6], q);
    if (e == cudaSuccess) e = cudaStreamSynchronize(q);
    st.refs_ms += w.ms(5, 6);
  }
  st.index_ms += w.ms(0, 1) + w.ms(2, 3);
  st.refs_ms += w.ms(3, 4);
  if (e != cudaSuccess) { ctx->err = std::string("lb2_syms_index: ") + cudaGetErrorString(e); return LB2_E_CUDA; }
  for (uint32_t i = 0; i < n; i++) {
    ids[i] = (uint32_t)s->objs.size();
    s->objs.push_back(objects[i]);
  }
  st.references = nrefs;
  st.arena_bytes = s->total;
  if (stats) *stats = st;
  return LB2_OK;
}

int lb2_syms_resolve(lb2_syms *s, const lb2_sym_job *jobs, uint32_t n_jobs, const uint32_t *scope, uint32_t n_scope,
                     const uint8_t *classes, uint32_t *counts, lb2_sym_miss *misses, uint32_t max_misses,
                     uint32_t *n_misses, lb2_syms_stats *stats) {
  if (!s) return LB2_E_ARG;
  lb2_ctx *ctx = s->ctx;
  const uint64_t n_obj = s->objs.size();
  if ((n_jobs && (!jobs || !counts)) || (n_scope && !scope) || (n_obj && !classes) || !n_misses || (max_misses && !misses)) {
    ctx->err = "NULL argument";
    return LB2_E_ARG;
  }
  for (uint32_t i = 0; i < n_scope; i++)
    if (scope[i] >= n_obj) { ctx->err = "lb2_syms_resolve: a scope entry is not an object id"; return LB2_E_ARG; }
  for (uint64_t i = 0; i < n_obj; i++)
    if (classes[i] > 2) { ctx->err = "lb2_syms_resolve: a class above 2"; return LB2_E_ARG; }
  std::vector<uint64_t> base(n_jobs + 1, 0);
  for (uint32_t j = 0; j < n_jobs; j++) {
    if (jobs[j].obj >= n_obj || jobs[j].scope_off > n_scope || jobs[j].scope_len > n_scope - jobs[j].scope_off) {
      ctx->err = "lb2_syms_resolve: a job outside the objects or the scope array";
      return LB2_E_ARG;
    }
    base[j + 1] = base[j] + s->objs[jobs[j].obj].nrefs;
  }
  lb2_syms_stats st{};
  *n_misses = 0;
  if (n_jobs) memset(counts, 0, 12ull * n_jobs);
  if (!n_jobs) { if (stats) *stats = st; return LB2_OK; }
  CK(cudaSetDevice(ctx->device));
  const uint64_t ob = sizeof(lb2_sym_object) * n_obj, jb = sizeof(lb2_sym_job) * n_jobs, bb = 8 * ((uint64_t)n_jobs + 1),
                 sb = 4ull * n_scope, cb = 12ull * n_jobs, mb = sizeof(lb2_sym_miss) * (uint64_t)max_misses;
  uint64_t o[8] = {0};  // offsets: objects, jobs, base, scope, classes, counts + n_miss + lookups, misses, end
  const uint64_t sz[7] = {ob, jb, bb, sb, n_obj, cb + 16, mb};
  for (int k = 0; k < 7; k++) o[k + 1] = (o[k] + sz[k] + 15) & ~15ull;
  SymScratch w(o[7]);
  cudaError_t &e = w.e;
  cudaStream_t q = ctx->stream;
  const void *src[5] = {s->objs.data(), jobs, base.data(), scope, classes};
  for (int k = 0; k < 5; k++)
    if (e == cudaSuccess && sz[k]) e = cudaMemcpyAsync(w.d + o[k], src[k], sz[k], cudaMemcpyHostToDevice, q);
  if (e == cudaSuccess) e = cudaMemsetAsync(w.d + o[5], 0, cb + 16, q);
  st.bytes_up = ob + jb + bb + sb + n_obj;
  uint32_t *d_counts = reinterpret_cast<uint32_t *>(w.d + o[5]), *d_nmiss = d_counts + 3ull * n_jobs;
  unsigned long long *d_lookups = reinterpret_cast<unsigned long long *>(w.d + ((o[5] + cb + 4 + 7) & ~7ull));
  if (e == cudaSuccess) e = cudaEventRecord(w.ev[0], q);
  if (e == cudaSuccess) {
    launch_syms_resolve(w.d + o[0], reinterpret_cast<const elfs::Job *>(w.d + o[1]), reinterpret_cast<const uint64_t *>(w.d + o[2]),
                        n_jobs, base[n_jobs], reinterpret_cast<const uint32_t *>(w.d + o[3]), w.d + o[4], d_counts,
                        reinterpret_cast<elfs::Miss *>(w.d + o[6]), max_misses, d_nmiss, d_lookups, q);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaEventRecord(w.ev[1], q);
  unsigned long long lookups = 0;
  if (e == cudaSuccess) e = cudaMemcpyAsync(counts, d_counts, cb, cudaMemcpyDeviceToHost, q);
  if (e == cudaSuccess) e = cudaMemcpyAsync(n_misses, d_nmiss, 4, cudaMemcpyDeviceToHost, q);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&lookups, d_lookups, 8, cudaMemcpyDeviceToHost, q);
  if (e == cudaSuccess) e = cudaStreamSynchronize(q);
  st.bytes_down = cb + 12;
  const uint32_t got = *n_misses < max_misses ? *n_misses : max_misses;
  if (e == cudaSuccess && got) e = cudaMemcpy(misses, w.d + o[6], sizeof(lb2_sym_miss) * (uint64_t)got, cudaMemcpyDeviceToHost);
  st.bytes_down += sizeof(lb2_sym_miss) * (uint64_t)got;
  st.resolve_ms = w.ms(0, 1);
  if (e != cudaSuccess) { ctx->err = std::string("lb2_syms_resolve: ") + cudaGetErrorString(e); return LB2_E_CUDA; }
  st.references = base[n_jobs];
  st.lookups = lookups;
  st.arena_bytes = s->total;
  if (stats) *stats = st;
  if (*n_misses > max_misses) { ctx->err = "lb2_syms_resolve: more misses than max_misses (*n_misses needed)"; return LB2_E_CAPACITY; }
  return LB2_OK;
}

int lb2_syms_names(lb2_syms *s, const lb2_sym_job *jobs, uint32_t n_jobs, const lb2_sym_miss *misses, uint32_t n,
                   uint64_t *offsets, void *h_pool, uint64_t pool_cap, uint64_t *pool_bytes, lb2_syms_stats *stats) {
  if (!s) return LB2_E_ARG;
  lb2_ctx *ctx = s->ctx;
  if ((n_jobs && !jobs) || (n && (!misses || !offsets)) || !pool_bytes || (pool_cap && !h_pool)) {
    ctx->err = "NULL argument";
    return LB2_E_ARG;
  }
  for (uint32_t j = 0; j < n_jobs; j++)
    if (jobs[j].obj >= s->objs.size()) { ctx->err = "lb2_syms_names: a job outside the objects"; return LB2_E_ARG; }
  for (uint32_t i = 0; i < n; i++)
    if (misses[i].job >= n_jobs || misses[i].ref >= s->objs[jobs[misses[i].job].obj].nrefs) {
      ctx->err = "lb2_syms_names: a miss outside its job's references";
      return LB2_E_ARG;
    }
  lb2_syms_stats st{};
  *pool_bytes = 0;
  if (!n) { if (stats) *stats = st; return LB2_OK; }
  CK(cudaSetDevice(ctx->device));
  const uint64_t ob = sizeof(lb2_sym_object) * s->objs.size(), jb = sizeof(lb2_sym_job) * n_jobs,
                 mb = sizeof(lb2_sym_miss) * (uint64_t)n, lb = 8ull * n;
  const uint64_t o1 = (ob + 15) & ~15ull, o2 = (o1 + jb + 15) & ~15ull, o3 = (o2 + mb + 15) & ~15ull, o4 = o3 + lb;
  SymScratch w(o4);
  cudaError_t &e = w.e;
  cudaStream_t q = ctx->stream;
  if (e == cudaSuccess) e = cudaMemcpyAsync(w.d, s->objs.data(), ob, cudaMemcpyHostToDevice, q);
  if (e == cudaSuccess && jb) e = cudaMemcpyAsync(w.d + o1, jobs, jb, cudaMemcpyHostToDevice, q);
  if (e == cudaSuccess) e = cudaMemcpyAsync(w.d + o2, misses, mb, cudaMemcpyHostToDevice, q);
  uint64_t *d_len = reinterpret_cast<uint64_t *>(w.d + o3);
  const elfs::Job *d_jobs = reinterpret_cast<const elfs::Job *>(w.d + o1);
  const elfs::Miss *d_miss = reinterpret_cast<const elfs::Miss *>(w.d + o2);
  if (e == cudaSuccess) { launch_syms_names(w.d, d_jobs, d_miss, n, d_len, nullptr, q); e = cudaGetLastError(); }
  if (e == cudaSuccess) e = cudaMemcpyAsync(offsets, d_len, lb, cudaMemcpyDeviceToHost, q);
  if (e == cudaSuccess) e = cudaStreamSynchronize(q);
  st.bytes_up += ob + jb + mb;
  st.bytes_down += lb;
  uint64_t total = 0;
  if (e == cudaSuccess)
    for (uint32_t i = 0; i < n; i++) {
      const uint64_t l = offsets[i];
      offsets[i] = total;
      total += l;
    }
  *pool_bytes = total;
  const bool fits = total <= pool_cap;
  uint8_t *d_pool = nullptr;
  if (e == cudaSuccess && fits) e = cudaMalloc(&d_pool, total);
  if (e == cudaSuccess && fits) e = cudaMemcpyAsync(d_len, offsets, lb, cudaMemcpyHostToDevice, q);
  if (e == cudaSuccess && fits) { launch_syms_names(w.d, d_jobs, d_miss, n, d_len, d_pool, q); e = cudaGetLastError(); }
  if (e == cudaSuccess && fits) e = cudaMemcpyAsync(h_pool, d_pool, total, cudaMemcpyDeviceToHost, q);
  if (e == cudaSuccess && fits) e = cudaStreamSynchronize(q);
  cudaFree(d_pool);
  if (fits) {
    st.bytes_up += lb;
    st.bytes_down += total;
  }
  if (e != cudaSuccess) { ctx->err = std::string("lb2_syms_names: ") + cudaGetErrorString(e); return LB2_E_CUDA; }
  if (stats) *stats = st;
  if (!fits) { ctx->err = "lb2_syms_names: the strings exceed pool_cap (*pool_bytes needed)"; return LB2_E_CAPACITY; }
  return LB2_OK;
}

int lb2_syms_find(lb2_syms *s, const lb2_sym_query *queries, uint32_t n, const uint32_t *scope, uint32_t n_scope,
                  const void *h_names, uint64_t names_bytes, lb2_sym_found *found, lb2_syms_stats *stats) {
  if (!s) return LB2_E_ARG;
  lb2_ctx *ctx = s->ctx;
  const uint64_t n_obj = s->objs.size();
  if ((n && (!queries || !found)) || (n_scope && !scope) || (names_bytes && !h_names)) {
    ctx->err = "NULL argument";
    return LB2_E_ARG;
  }
  for (uint32_t i = 0; i < n_scope; i++)
    if (scope[i] >= n_obj) { ctx->err = "lb2_syms_find: a scope entry is not an object id"; return LB2_E_ARG; }
  for (uint32_t q = 0; q < n; q++)
    if (queries[q].scope_off > n_scope || queries[q].scope_len > n_scope - queries[q].scope_off ||
        queries[q].name_off > names_bytes || queries[q].name_len > names_bytes - queries[q].name_off) {
      ctx->err = "lb2_syms_find: a query outside the scope array or the name pool";
      return LB2_E_ARG;
    }
  lb2_syms_stats st{};
  if (!n) { if (stats) *stats = st; return LB2_OK; }
  CK(cudaSetDevice(ctx->device));
  const uint64_t ob = sizeof(lb2_sym_object) * n_obj, qb = sizeof(lb2_sym_query) * (uint64_t)n, sb = 4ull * n_scope,
                 fb = sizeof(lb2_sym_found) * (uint64_t)n;
  uint64_t o[6] = {0};  // offsets: objects, queries, scope, names, found, end
  const uint64_t sz[5] = {ob, qb, sb, names_bytes, fb};
  for (int k = 0; k < 5; k++) o[k + 1] = (o[k] + sz[k] + 15) & ~15ull;
  SymScratch w(o[5]);
  cudaError_t &e = w.e;
  cudaStream_t q = ctx->stream;
  const void *src[4] = {s->objs.data(), queries, scope, h_names};
  for (int k = 0; k < 4; k++)
    if (e == cudaSuccess && sz[k]) e = cudaMemcpyAsync(w.d + o[k], src[k], sz[k], cudaMemcpyHostToDevice, q);
  st.bytes_up = ob + qb + sb + names_bytes;
  if (e == cudaSuccess) e = cudaEventRecord(w.ev[0], q);
  if (e == cudaSuccess) {
    launch_syms_find(w.d + o[0], reinterpret_cast<const elfs::Query *>(w.d + o[1]), n,
                     reinterpret_cast<const uint32_t *>(w.d + o[2]), w.d + o[3], reinterpret_cast<elfs::Found *>(w.d + o[4]), q);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaEventRecord(w.ev[1], q);
  if (e == cudaSuccess) e = cudaMemcpyAsync(found, w.d + o[4], fb, cudaMemcpyDeviceToHost, q);
  if (e == cudaSuccess) e = cudaStreamSynchronize(q);
  st.bytes_down = fb;
  st.resolve_ms = w.ms(0, 1);
  if (e != cudaSuccess) { ctx->err = std::string("lb2_syms_find: ") + cudaGetErrorString(e); return LB2_E_CUDA; }
  st.references = n;
  st.arena_bytes = s->total;
  if (stats) *stats = st;
  return LB2_OK;
}

}  // extern "C"
