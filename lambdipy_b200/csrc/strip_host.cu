// strip_host.cu -- lb2_strip_host: arenas in host memory.  Zero-copy (the kernels work on the pinned arenas through
// their device mapping), copy-engine (LB2_HOST_DMA=1) and staged (pageable arenas or LB2_HOST_ZEROCOPY=0).
#include "lb2_host.cuh"

// The slots of the staged and copy-engine pipelines: chunk k runs in slot k % NS.
constexpr int NS = 3;
struct HostSlots {
  struct Slot {
    Workspace ws;
    cudaStream_t stream = nullptr;
    uint8_t *d_in = nullptr, *d_out = nullptr;
    uint64_t cap_in = 0, cap_out = 0;
    cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_d2h[2] = {nullptr, nullptr};
  } slot[NS];
};

void host_slots_free(HostSlots *h) {
  if (!h) return;
  for (auto &sl : h->slot) {
    ws_free(sl.ws);
    cudaFree(sl.d_in); cudaFree(sl.d_out);
    if (sl.stream) cudaStreamDestroy(sl.stream);
    for (auto &e : sl.ev_h2d) if (e) cudaEventDestroy(e);
    for (auto &e : sl.ev_d2h) if (e) cudaEventDestroy(e);
  }
  delete h;
}

// The slots with their streams and events, created on first use.
static int host_slots_prepare(lb2_ctx *ctx) {
  if (!ctx->host) ctx->host = new HostSlots();
  for (auto &sl : ctx->host->slot) {
    if (sl.stream) continue;
    CK(cudaStreamCreateWithFlags(&sl.stream, cudaStreamNonBlocking));
    for (auto &e : sl.ev_h2d) CK(cudaEventCreate(&e));
    for (auto &e : sl.ev_d2h) CK(cudaEventCreate(&e));
  }
  return LB2_OK;
}

// ---- host buffers, pinned and mapped: plan over the mapping, upload only what is kept, compact in HBM ----------
// The copy engines move more bytes per second over PCIe than SM loads/stores on mapped host memory (what the
// zero-copy path gets; tools/pcie_probe.cu measures both).  So, per chunk of whole files (<= LB2_CHUNK_MB of
// arena span, three slots rotating):
//   1. plan + scan run on the host-mapped input: only headers, names and notes cross the bus; the kernel also
//      lists the input ranges its copy extents read (small files whole, neighbours merged);
//   2. those ranges are uploaded by the copy engine into a device slot laid out like the host arena -- dropped
//      sections (.symtab/.strtab/.debug_*) still never cross the bus;
//   3. the compaction kernel runs HBM -> HBM (tile sources inside the host mapping are rebased onto the slot);
//   4. one DMA brings the chunk's output down.
// The plan of chunk k+1 is queued before the host waits for chunk k's plan results, so the engines stay busy.
static int strip_host_dma(lb2_ctx *ctx, const uint8_t *h_in, const uint8_t *d_in_alias, const uint64_t *h_in_off, const uint64_t *h_in_sizes,
                          uint32_t n_files, uint8_t *h_out, uint64_t out_capacity, uint64_t *h_out_off, uint64_t *h_out_sizes,
                          int32_t *h_status, uint32_t flags, lb2_stats *stats) {
  const uint64_t chunk_bytes = env_u64("LB2_CHUNK_MB", 256) << 20;
  lb2_stats total;
  memset(&total, 0, sizeof total);
  total.n_files = n_files;
  const std::vector<Chunk> chunks = split_chunks(h_in_off, n_files, chunk_bytes);
  int rc = host_slots_prepare(ctx);
  if (rc) return rc;
  HostSlots::Slot *slot = ctx->host->slot;
  uint64_t out_base = 0;
  std::vector<uint64_t> rel_off, coff;
  auto plan = [&](size_t ci) -> int {
    auto &sl = slot[ci % NS];
    const Chunk &c = chunks[ci];
    const uint32_t n = c.f1 - c.f0;
    if (ci >= (size_t)NS) {  // the slot's previous occupant must be fully downloaded
      CK(cudaEventSynchronize(sl.ev_d2h[1]));
      float a = 0, b = 0;
      cudaEventElapsedTime(&a, sl.ev_h2d[0], sl.ev_h2d[1]);
      cudaEventElapsedTime(&b, sl.ev_d2h[0], sl.ev_d2h[1]);
      total.h2d_ms += a; total.d2h_ms += b;
    }
    rel_off.resize(n + 1);
    for (uint32_t i = 0; i <= n; i++) rel_off[i] = h_in_off[c.f0 + i] - c.in_base;
    return enqueue_batch(ctx, sl.ws, d_in_alias + c.in_base, rel_off.data(), h_in_sizes ? h_in_sizes + c.f0 : nullptr, n, nullptr, 0, flags,
                         sl.stream, false, true, true);
  };
  auto move = [&](size_t ci) -> int {
    auto &sl = slot[ci % NS];
    const Chunk &c = chunks[ci];
    const uint32_t n = c.f1 - c.f0;
    lb2_stats st;
    coff.resize(n + 1);
    int r = collect_batch(ctx, sl.ws, coff.data(), h_out_sizes + c.f0, h_status + c.f0, &st);
    if (r) return r;
    const uint64_t bytes = coff[n];
    if (out_base + bytes > out_capacity) { ctx->err = "host output arena too small"; total.out_bytes_needed = out_base + bytes; return LB2_E_CAPACITY; }
    if (sl.cap_in < c.in_span + 256)
      CK(regrow(&sl.d_in, sl.cap_in, std::max<uint64_t>(c.in_span + 256, std::min<uint64_t>(chunk_bytes, 64ull << 20))));
    if (sl.cap_out < bytes + 256) CK(regrow(&sl.d_out, sl.cap_out, std::max<uint64_t>(bytes + (1u << 20), c.in_span + (8u << 20))));
    // upload what the copy extents read
    const BatchCounters &bc = *sl.ws.h_ctr;
    CK(cudaEventRecord(sl.ev_h2d[0], sl.stream));
    if (bc.ranges_overflow || bc.n_ranges > sl.ws.cap_ranges) {
      CK(cudaMemcpyAsync(sl.d_in, h_in + c.in_base, h_in_off[c.f1] - c.in_base, cudaMemcpyHostToDevice, sl.stream));
      total.h2d_bytes += h_in_off[c.f1] - c.in_base;
    } else {
      // the kernel appended the ranges in no particular order: sort, fuse neighbours (files are 256-byte
      // padded, so runs of small files become one transfer), one DMA per fused range
      UpRange *rg = sl.ws.h_ranges;
      std::sort(rg, rg + bc.n_ranges, [](const UpRange &x, const UpRange &y) { return x.off < y.off; });
      uint64_t rs = 0, re = 0;
      auto flush = [&]() -> int {
        if (re <= rs) return LB2_OK;
        if (re > c.in_span) { ctx->err = "upload range outside the chunk"; return LB2_E_STATE; }
        CK(cudaMemcpyAsync(sl.d_in + rs, h_in + c.in_base + rs, re - rs, cudaMemcpyHostToDevice, sl.stream));
        total.h2d_bytes += re - rs;
        return LB2_OK;
      };
      for (uint32_t k = 0; k < bc.n_ranges; k++) {
        const uint64_t o = rg[k].off, e = rg[k].off + rg[k].len;
        if (re > rs && o <= re + 8192) { if (e > re) re = e; }
        else { int fr = flush(); if (fr) return fr; rs = o; re = e; }
      }
      int fr = flush();
      if (fr) return fr;
    }
    CK(cudaEventRecord(sl.ev_h2d[1], sl.stream));
    // compaction on the device copy
    CompactArgs ca;
    ca.tiles = sl.ws.d_tiles; ca.ctr = sl.ws.d_ctr; ca.out_off = sl.ws.d_out_off; ca.out = sl.d_out;
    ca.rebase_lo = reinterpret_cast<uint64_t>(d_in_alias + c.in_base);
    ca.rebase_len = c.in_span;
    ca.rebase_delta = reinterpret_cast<uint64_t>(sl.d_in) - ca.rebase_lo;
    CK(cudaEventRecord(sl.ws.ev[1], sl.stream));
    enqueue_compact(ctx, ca, sl.stream);
    CK(cudaEventRecord(sl.ws.ev[2], sl.stream));
    CK(cudaEventRecord(sl.ev_d2h[0], sl.stream));
    if (bytes) CK(cudaMemcpyAsync(h_out + out_base, sl.d_out, bytes, cudaMemcpyDeviceToHost, sl.stream));
    total.d2h_bytes += bytes;
    total.h2d_bytes += st.header_bytes;   // what the plan kernel read through the mapping
    CK(cudaEventRecord(sl.ev_d2h[1], sl.stream));
    CK(cudaGetLastError());
    for (uint32_t i = 0; i < n; i++) h_out_off[c.f0 + i] = out_base + coff[i];
    out_base += bytes;
    st.compact_ms = 0;  // st is of the plan-only batch; the compaction times are read from the slots at the end
    add_stats(total, st);
    return LB2_OK;
  };
  for (size_t ci = 0; ci < chunks.size() && rc == LB2_OK; ci++) {
    rc = plan(ci);
    if (rc == LB2_OK && ci >= 1) rc = move(ci - 1);
  }
  if (rc == LB2_OK && !chunks.empty()) rc = move(chunks.size() - 1);
  for (int k = 0; k < NS; k++) {
    auto &sl = slot[k];
    cudaStreamSynchronize(sl.stream);
    sl.ws.in_flight = false;
    if ((size_t)k < chunks.size()) {
      float a = 0, b = 0, cms = 0;
      if (cudaEventElapsedTime(&a, sl.ev_h2d[0], sl.ev_h2d[1]) == cudaSuccess) total.h2d_ms += a;
      if (cudaEventElapsedTime(&b, sl.ev_d2h[0], sl.ev_d2h[1]) == cudaSuccess) total.d2h_ms += b;
      if (cudaEventElapsedTime(&cms, sl.ws.ev[1], sl.ws.ev[2]) == cudaSuccess) total.compact_ms += cms;  // (last chunk of each slot only)
    }
  }
  cudaGetLastError();
  h_out_off[n_files] = out_base;
  if (total.out_bytes_needed == 0) total.out_bytes_needed = out_base;
  if (stats) *stats = total;
  return rc;
}

extern "C" {

int lb2_strip_host(lb2_ctx *ctx, const void *h_in_v, const uint64_t *h_in_off, const uint64_t *h_in_sizes, uint32_t n_files,
                   void *h_out_v, uint64_t out_capacity, uint64_t *h_out_off, uint64_t *h_out_sizes, int32_t *h_status,
                   uint32_t flags, lb2_stats *stats) {
  if (!ctx || !h_in_v || !h_in_off || !h_out_v || !h_out_off || !h_out_sizes || !h_status) { if (ctx) ctx->err = "NULL argument"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  const uint8_t *h_in = static_cast<const uint8_t *>(h_in_v);
  uint8_t *h_out = static_cast<uint8_t *>(h_out_v);
  // Zero-copy path: when both arenas are pinned and mapped into the device address space the
  // kernels work on them directly over PCIe -- the plan kernel pulls only headers, the compaction
  // kernel pulls only the KEPT extents and pushes the stripped files straight into host memory.
  // Dropped sections (.symtab/.strtab/.debug_*) never cross the bus, uploads and downloads run
  // concurrently in both directions, and nothing has to fit in HBM.
  if (env_u64("LB2_HOST_ZEROCOPY", 1) && n_files) {
    void *d_in_alias = nullptr, *d_out_alias = nullptr;
    cudaPointerAttributes ai, ao;
    const bool ok = cudaPointerGetAttributes(&ai, h_in) == cudaSuccess && ai.type == cudaMemoryTypeHost &&
                    cudaPointerGetAttributes(&ao, h_out) == cudaSuccess && ao.type == cudaMemoryTypeHost &&
                    cudaHostGetDevicePointer(&d_in_alias, const_cast<uint8_t *>(h_in), 0) == cudaSuccess &&
                    cudaHostGetDevicePointer(&d_out_alias, h_out, 0) == cudaSuccess;
    cudaGetLastError();  // clear "invalid value" from probing pageable memory
    if (ok && env_u64("LB2_HOST_DMA", 0)) {
      // opt-in (LB2_HOST_DMA=1): plan over the mapping, copy-engine transfers of the kept ranges, compaction in HBM.
      // The copy engines' edge over SM loads/stores is largely eaten by the per-chunk plan -> host -> DMA hand-over.
      return strip_host_dma(ctx, h_in, static_cast<const uint8_t *>(d_in_alias), h_in_off, h_in_sizes, n_files, h_out, out_capacity,
                            h_out_off, h_out_sizes, h_status, flags, stats);
    }
    if (ok) {
      int rc = enqueue_batch(ctx, ctx->ws, static_cast<const uint8_t *>(d_in_alias), h_in_off, h_in_sizes, n_files,
                             static_cast<uint8_t *>(d_out_alias), out_capacity, flags, ctx->stream, true);
      if (rc) return rc;
      lb2_stats st;
      rc = collect_batch(ctx, ctx->ws, h_out_off, h_out_sizes, h_status, &st);
      st.h2d_bytes = st.copy_bytes + st.header_bytes;   // pulled by the kernels through the mapping
      st.d2h_bytes = st.out_bytes;
      if (stats) *stats = st;
      return rc;
    }
  }
  const uint64_t chunk_bytes = env_u64("LB2_CHUNK_MB", 256) << 20;
  lb2_stats total;
  memset(&total, 0, sizeof total);
  total.n_files = n_files;
  const std::vector<Chunk> chunks = split_chunks(h_in_off, n_files, chunk_bytes);
  int rc = host_slots_prepare(ctx);
  if (rc) return rc;
  HostSlots::Slot *slot = ctx->host->slot;
  std::vector<uint64_t> rel_off;
  uint64_t out_base = 0;  // running 256-aligned position in h_out

  auto finish = [&](size_t ci) -> int {
    auto &sl = slot[ci % NS];
    const Chunk &c = chunks[ci];
    const uint32_t n = c.f1 - c.f0;
    // wait for plan+scan (+compact, same stream) and learn the chunk's output size
    lb2_stats st;
    std::vector<uint64_t> coff(n + 1);
    int r = collect_batch(ctx, sl.ws, coff.data(), h_out_sizes + c.f0, h_status + c.f0, &st);
    if (r == LB2_E_CAPACITY) {  // device-side output slot too small: enlarge and redo this chunk
      std::vector<uint64_t> ro(n + 1);
      for (uint32_t i = 0; i <= n; i++) ro[i] = h_in_off[c.f0 + i] - c.in_base;
      r = redo_grown(ctx, sl.ws, sl.d_in, ro.data(), h_in_sizes ? h_in_sizes + c.f0 : nullptr, n, sl.d_out, sl.cap_out, flags, sl.stream,
                     coff.data(), h_out_sizes + c.f0, h_status + c.f0, &st);
    }
    if (r) return r;
    const uint64_t bytes = coff[n];
    if (out_base + bytes > out_capacity) { ctx->err = "host output arena too small"; total.out_bytes_needed = out_base + bytes; return LB2_E_CAPACITY; }
    CK(cudaEventRecord(sl.ev_d2h[0], sl.stream));
    if (bytes) CK(cudaMemcpyAsync(h_out + out_base, sl.d_out, bytes, cudaMemcpyDeviceToHost, sl.stream));
    total.d2h_bytes += bytes;
    CK(cudaEventRecord(sl.ev_d2h[1], sl.stream));
    for (uint32_t i = 0; i < n; i++) h_out_off[c.f0 + i] = out_base + coff[i];
    out_base += bytes;
    add_stats(total, st);
    return LB2_OK;
  };
  auto reap_copy_times = [&](size_t ci) {
    auto &sl = slot[ci % NS];
    cudaEventSynchronize(sl.ev_d2h[1]);
    float a = 0, b = 0;
    cudaEventElapsedTime(&a, sl.ev_h2d[0], sl.ev_h2d[1]);
    cudaEventElapsedTime(&b, sl.ev_d2h[0], sl.ev_d2h[1]);
    total.h2d_ms += a; total.d2h_ms += b;
  };

  for (size_t ci = 0; ci < chunks.size() && rc == LB2_OK; ci++) {
    auto &sl = slot[ci % NS];
    const Chunk &c = chunks[ci];
    const uint32_t n = c.f1 - c.f0;
    if (ci >= (size_t)NS) reap_copy_times(ci - NS);  // slot is free once its D2H finished
    if (sl.cap_in < c.in_span + 256)
      CK(regrow(&sl.d_in, sl.cap_in, std::max<uint64_t>(c.in_span + 256, std::min<uint64_t>(chunk_bytes, 64ull << 20))));
    const uint64_t want_out = c.in_span + (uint64_t)n * 4096 + (8u << 20);
    if (sl.cap_out < want_out) CK(regrow(&sl.d_out, sl.cap_out, want_out));
    CK(cudaEventRecord(sl.ev_h2d[0], sl.stream));
    CK(cudaMemcpyAsync(sl.d_in, h_in + c.in_base, h_in_off[c.f1] - c.in_base, cudaMemcpyHostToDevice, sl.stream));
    total.h2d_bytes += h_in_off[c.f1] - c.in_base;
    CK(cudaEventRecord(sl.ev_h2d[1], sl.stream));
    rel_off.resize(n + 1);
    for (uint32_t i = 0; i <= n; i++) rel_off[i] = h_in_off[c.f0 + i] - c.in_base;
    rc = enqueue_batch(ctx, sl.ws, sl.d_in, rel_off.data(), h_in_sizes ? h_in_sizes + c.f0 : nullptr, n, sl.d_out, sl.cap_out, flags, sl.stream, true);
    if (rc) break;
    // with the next chunk's upload and kernels queued, turn to the previous chunk's download
    if (ci >= 1) rc = finish(ci - 1);
  }
  if (rc == LB2_OK && !chunks.empty()) rc = finish(chunks.size() - 1);
  for (size_t ci = chunks.size() >= (size_t)NS ? chunks.size() - NS : 0; ci < chunks.size(); ci++) reap_copy_times(ci);
  for (int k = 0; k < NS; k++) { cudaStreamSynchronize(slot[k].stream); slot[k].ws.in_flight = false; }
  h_out_off[n_files] = out_base;
  if (total.out_bytes_needed == 0) total.out_bytes_needed = out_base;
  if (stats) *stats = total;
  return rc;
}

}  // extern "C"
