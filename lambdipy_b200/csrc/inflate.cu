// inflate.cu -- kernels of the speculative parallel DEFLATE decoder behind lb2_inflate_* and lb2_unzip_* (api.cu).
// The decoding logic is inflate_core.cuh; the kernels only map it onto the GPU.  Every kernel works from a table of
// streams (the gzip reader's one stream is the one-entry case), and every bit a span reads is bounded by its own stream:
//   find     one warp per (stream, nominal span k >= 1): the lanes test 32 consecutive bit positions at a time and the
//            lowest passing one is the span's candidate;
//   count    one thread per span, tables in shared memory: decode without writing, record the end key and length;
//   decode   one thread per confirmed span: the same walk, writing the u16 arena;
//   table    one thread per seek-table span (exact stop): the decode walk, also writing each span's result, which the
//            host checks before it trusts the table;
//   window   one CTA per stream walks its spans in order and makes the last 32 KB of each final (the next span's window);
//   resolve  one CTA per span makes the rest final, reading marker values from the windows;
//   small    (zip reader) one thread per stream of at most one span: the byte-output walk, straight into the output;
//   copy     (zip reader) one warp per STORED member.
#include "lb2_common.cuh"
#include "copy_device.cuh"
#include "inflate_core.cuh"

namespace lb2 {
namespace {
using namespace ifl;

constexpr int FIND_THREADS = 64;  // two spans per CTA
constexpr int SPAN_THREADS = 32;
constexpr int WINDOW_THREADS = 1024;
constexpr int RESOLVE_THREADS = 256;

__global__ void __launch_bounds__(FIND_THREADS) lb2_inflate_find_kernel(const uint8_t *base, uint64_t span,
                                                                         const FindJob *jobs, uint32_t n_jobs, uint64_t *cand) {
  extern __shared__ __align__(16) uint8_t smem[];
  HdrScratch &s = reinterpret_cast<HdrScratch *>(smem)[threadIdx.x];
  const uint32_t j = blockIdx.x * (FIND_THREADS / 32) + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (j >= n_jobs) return;  // the whole warp
  const FindJob fj = jobs[j];
  const uint8_t *in = base + fj.in_off;
  const uint64_t n = fj.in_n, k = fj.k;
  const uint64_t from = k * span * 8;
  const uint64_t to = ((k + 1) * span < n ? (k + 1) * span : n) * 8;
  uint64_t found = KEY_NONE;
  for (uint64_t base = from; base < to; base += 32) {
    const uint64_t p = base + lane;
    const uint64_t key = p < to ? candidate_at(in, n, p, s) : KEY_NONE;
    const unsigned m = __ballot_sync(0xffffffffu, key != KEY_NONE);
    if (m) {
      found = __shfl_sync(0xffffffffu, key, __ffs(m) - 1);
      break;
    }
  }
  if (lane == 0) cand[j] = found;
}

__global__ void __launch_bounds__(SPAN_THREADS) lb2_inflate_count_kernel(const uint8_t *in, const SpanJob *jobs, uint32_t n_jobs,
                                                                          SpanResult *res) {
  extern __shared__ __align__(16) uint8_t smem[];
  DecodeState &st = reinterpret_cast<DecodeState *>(smem)[threadIdx.x];
  const uint32_t i = blockIdx.x * SPAN_THREADS + threadIdx.x;
  if (i >= n_jobs) return;
  const SpanJob j = jobs[i];
  SpanResult r;
  decode_span<false>(in + j.in_off, j.in_n, j, st, (uint16_t *)nullptr, r);
  res[i] = r;
}

__global__ void __launch_bounds__(SPAN_THREADS) lb2_inflate_decode_kernel(const uint8_t *in, const SpanJob *jobs, uint32_t n_jobs,
                                                                           uint16_t *arena, int32_t *err) {
  extern __shared__ __align__(16) uint8_t smem[];
  DecodeState &st = reinterpret_cast<DecodeState *>(smem)[threadIdx.x];
  const uint32_t i = blockIdx.x * SPAN_THREADS + threadIdx.x;
  if (i >= n_jobs) return;
  const SpanJob j = jobs[i];
  SpanResult r;
  decode_span<true>(in + j.in_off, j.in_n, j, st, arena + j.out_off, r);
  if (r.status != ifl::ST_OK) atomicExch(err + j.member, r.status);
}

__global__ void __launch_bounds__(SPAN_THREADS) lb2_inflate_table_decode_kernel(const uint8_t *in, const SpanJob *jobs,
                                                                                 uint32_t n_jobs, uint16_t *arena,
                                                                                 SpanResult *res) {
  extern __shared__ __align__(16) uint8_t smem[];
  DecodeState &st = reinterpret_cast<DecodeState *>(smem)[threadIdx.x];
  const uint32_t i = blockIdx.x * SPAN_THREADS + threadIdx.x;
  if (i >= n_jobs) return;
  const SpanJob j = jobs[i];
  SpanResult r;
  decode_span<true>(in + j.in_off, j.in_n, j, st, arena + j.out_off, r);
  res[i] = r;
}

constexpr int32_t ERR_WINDOW = -100;  // a marker points before the stream start

// CTA b: the spans first[b] .. first[b + 1] - 1 of one stream
__global__ void __launch_bounds__(WINDOW_THREADS) lb2_inflate_window_kernel(const uint16_t *arena, uint8_t *out,
                                                                             const SpanJob *jobs, const uint32_t *first,
                                                                             int32_t *err) {
  bool bad = false;
  const uint32_t jb = first[blockIdx.x], je = first[blockIdx.x + 1];
  for (uint32_t j = jb; j < je; j++) {
    const uint64_t off = jobs[j].out_off, len = jobs[j].out_len, base = jobs[j].out_base;
    for (uint64_t i = (len > 32768 ? len - 32768 : 0) + threadIdx.x; i < len; i += WINDOW_THREADS)
      bad |= !resolve_value(arena[off + i], off, out, out[off + i], base);
    __syncthreads();
  }
  if (bad && je > jb) atomicExch(err + jobs[jb].member, ERR_WINDOW);
}

__global__ void __launch_bounds__(RESOLVE_THREADS) lb2_inflate_resolve_kernel(const uint16_t *arena, uint8_t *out,
                                                                               const SpanJob *jobs, int32_t *err) {
  const SpanJob &j = jobs[blockIdx.x];
  const uint64_t off = j.out_off, len = j.out_len, base = j.out_base;
  bool bad = false;
  for (uint64_t i = threadIdx.x; i + 32768 < len; i += RESOLVE_THREADS)
    bad |= !resolve_value(arena[off + i], off, out, out[off + i], base);
  if (bad) atomicExch(err + j.member, ERR_WINDOW);
}

// a member of at most one span, decoded whole into out[j.out_off .. + j.out_len): its status is its own
__global__ void __launch_bounds__(SPAN_THREADS) lb2_unzip_small_kernel(const uint8_t *in, const SpanJob *jobs, uint32_t n_jobs,
                                                                        uint8_t *out, int32_t *status) {
  extern __shared__ __align__(16) uint8_t smem[];
  DecodeState &st = reinterpret_cast<DecodeState *>(smem)[threadIdx.x];
  const uint32_t i = blockIdx.x * SPAN_THREADS + threadIdx.x;
  if (i >= n_jobs) return;
  const SpanJob j = jobs[i];
  SpanResult r;
  decode_span<true, uint8_t>(in + j.in_off, j.in_n, j, st, out + j.out_off, r);
  status[j.member] = member_status(r.status);
}

// one warp per STORED member, in tiles of the compaction kernels' byte mover
__global__ void __launch_bounds__(256) lb2_unzip_copy_kernel(const uint8_t *in, const Member *members, const uint32_t *idx,
                                                              uint32_t n, uint8_t *out) {
  const uint32_t w = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (w >= n) return;
  const Member m = members[idx[w]];
  const int lane = threadIdx.x & 31;
  for (uint64_t o = 0; o < m.out_len; o += TILE_BYTES) {
    const uint32_t len = (uint32_t)(m.out_len - o < TILE_BYTES ? m.out_len - o : TILE_BYTES);
    warp_copy_tile(in + m.in_off + o, out + m.out_off + o, len, lane);
  }
}

}  // namespace

void launch_inflate_find(const uint8_t *in, uint64_t span, const FindJob *jobs, uint32_t n_jobs, uint64_t *cand, cudaStream_t s) {
  if (!n_jobs) return;
  const uint32_t smem = FIND_THREADS * sizeof(HdrScratch);
  cudaFuncSetAttribute(lb2_inflate_find_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  lb2_inflate_find_kernel<<<(n_jobs + FIND_THREADS / 32 - 1) / (FIND_THREADS / 32), FIND_THREADS, smem, s>>>(in, span, jobs, n_jobs, cand);
}
void launch_inflate_count(const uint8_t *in, const SpanJob *jobs, uint32_t n_jobs, SpanResult *res, cudaStream_t s) {
  if (!n_jobs) return;
  const uint32_t smem = SPAN_THREADS * sizeof(DecodeState);
  cudaFuncSetAttribute(lb2_inflate_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  lb2_inflate_count_kernel<<<(n_jobs + SPAN_THREADS - 1) / SPAN_THREADS, SPAN_THREADS, smem, s>>>(in, jobs, n_jobs, res);
}
void launch_inflate_decode(const uint8_t *in, const SpanJob *jobs, uint32_t n_jobs, uint16_t *arena, int32_t *err, cudaStream_t s) {
  if (!n_jobs) return;
  const uint32_t smem = SPAN_THREADS * sizeof(DecodeState);
  cudaFuncSetAttribute(lb2_inflate_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  lb2_inflate_decode_kernel<<<(n_jobs + SPAN_THREADS - 1) / SPAN_THREADS, SPAN_THREADS, smem, s>>>(in, jobs, n_jobs, arena, err);
}
void launch_inflate_table_decode(const uint8_t *in, const SpanJob *jobs, uint32_t n_jobs, uint16_t *arena, SpanResult *res,
                                 cudaStream_t s) {
  if (!n_jobs) return;
  const uint32_t smem = SPAN_THREADS * sizeof(DecodeState);
  cudaFuncSetAttribute(lb2_inflate_table_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  lb2_inflate_table_decode_kernel<<<(n_jobs + SPAN_THREADS - 1) / SPAN_THREADS, SPAN_THREADS, smem, s>>>(in, jobs, n_jobs,
                                                                                                         arena, res);
}
void launch_inflate_resolve(const uint16_t *arena, uint8_t *out, const SpanJob *jobs, uint32_t n_jobs, const uint32_t *first,
                            uint32_t n_streams, int32_t *err, cudaStream_t s) {
  if (!n_jobs) return;
  lb2_inflate_window_kernel<<<n_streams, WINDOW_THREADS, 0, s>>>(arena, out, jobs, first, err);
  lb2_inflate_resolve_kernel<<<n_jobs, RESOLVE_THREADS, 0, s>>>(arena, out, jobs, err);
}
void launch_unzip_small(const uint8_t *in, const SpanJob *jobs, uint32_t n_jobs, uint8_t *out, int32_t *status, cudaStream_t s) {
  if (!n_jobs) return;
  const uint32_t smem = SPAN_THREADS * sizeof(DecodeState);
  cudaFuncSetAttribute(lb2_unzip_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  lb2_unzip_small_kernel<<<(n_jobs + SPAN_THREADS - 1) / SPAN_THREADS, SPAN_THREADS, smem, s>>>(in, jobs, n_jobs, out, status);
}
void launch_unzip_copy(const uint8_t *in, const Member *members, const uint32_t *idx, uint32_t n, uint8_t *out, cudaStream_t s) {
  if (!n) return;
  lb2_unzip_copy_kernel<<<(n + 7) / 8, 256, 0, s>>>(in, members, idx, n, out);
}

}  // namespace lb2
