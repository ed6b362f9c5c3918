// inflate.cu -- kernels of the speculative parallel DEFLATE decoder behind lb2_inflate_* (api.cu).  The decoding
// logic is inflate_core.cuh; the kernels only map it onto the GPU:
//   find     one warp per nominal span k >= 1: the lanes test 32 consecutive bit positions at a time and the lowest
//            passing one is the span's candidate;
//   count    one thread per span, tables in shared memory: decode without writing, record the end key and length;
//   decode   one thread per confirmed span: the same walk, writing the u16 arena;
//   window   one CTA walks the spans in order and makes the last 32 KB of each final (the next span's window);
//   resolve  one CTA per span makes the rest final, reading marker values from the windows.
#include "lb2_common.cuh"
#include "inflate_core.cuh"

namespace lb2 {
namespace {
using namespace ifl;

constexpr int FIND_THREADS = 64;  // two spans per CTA
constexpr int SPAN_THREADS = 32;
constexpr int WINDOW_THREADS = 1024;
constexpr int RESOLVE_THREADS = 256;

__global__ void __launch_bounds__(FIND_THREADS) lb2_inflate_find_kernel(const uint8_t *in, uint64_t n, uint64_t span,
                                                                         uint32_t n_spans, uint64_t *cand) {
  extern __shared__ __align__(16) uint8_t smem[];
  HdrScratch &s = reinterpret_cast<HdrScratch *>(smem)[threadIdx.x];
  const uint32_t k = blockIdx.x * (FIND_THREADS / 32) + threadIdx.x / 32 + 1;
  const int lane = threadIdx.x & 31;
  if (k >= n_spans) return;  // the whole warp
  const uint64_t from = (uint64_t)k * span * 8;
  const uint64_t to = ((uint64_t)(k + 1) * span < n ? (uint64_t)(k + 1) * span : n) * 8;
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
  if (lane == 0) cand[k] = found;
}

__global__ void __launch_bounds__(SPAN_THREADS) lb2_inflate_count_kernel(const uint8_t *in, uint64_t n, const SpanJob *jobs,
                                                                          uint32_t n_jobs, SpanResult *res) {
  extern __shared__ __align__(16) uint8_t smem[];
  DecodeState &st = reinterpret_cast<DecodeState *>(smem)[threadIdx.x];
  const uint32_t i = blockIdx.x * SPAN_THREADS + threadIdx.x;
  if (i >= n_jobs) return;
  SpanResult r;
  decode_span<false>(in, n, jobs[i], st, nullptr, r);
  res[i] = r;
}

__global__ void __launch_bounds__(SPAN_THREADS) lb2_inflate_decode_kernel(const uint8_t *in, uint64_t n, const SpanJob *jobs,
                                                                           uint32_t n_jobs, uint16_t *arena, int32_t *err) {
  extern __shared__ __align__(16) uint8_t smem[];
  DecodeState &st = reinterpret_cast<DecodeState *>(smem)[threadIdx.x];
  const uint32_t i = blockIdx.x * SPAN_THREADS + threadIdx.x;
  if (i >= n_jobs) return;
  const SpanJob j = jobs[i];
  SpanResult r;
  decode_span<true>(in, n, j, st, arena + j.out_off, r);
  if (r.status != ifl::ST_OK) atomicExch(err, r.status);
}

constexpr int32_t ERR_WINDOW = -100;  // a marker points before the stream start

__global__ void __launch_bounds__(WINDOW_THREADS) lb2_inflate_window_kernel(const uint16_t *arena, uint8_t *out,
                                                                             const SpanJob *jobs, uint32_t n_jobs, int32_t *err) {
  bool bad = false;
  for (uint32_t j = 0; j < n_jobs; j++) {
    const uint64_t off = jobs[j].out_off, len = jobs[j].out_len;
    for (uint64_t i = (len > 32768 ? len - 32768 : 0) + threadIdx.x; i < len; i += WINDOW_THREADS)
      bad |= !resolve_value(arena[off + i], off, out, out[off + i]);
    __syncthreads();
  }
  if (bad) atomicExch(err, ERR_WINDOW);
}

__global__ void __launch_bounds__(RESOLVE_THREADS) lb2_inflate_resolve_kernel(const uint16_t *arena, uint8_t *out,
                                                                               const SpanJob *jobs, int32_t *err) {
  const uint64_t off = jobs[blockIdx.x].out_off, len = jobs[blockIdx.x].out_len;
  bool bad = false;
  for (uint64_t i = threadIdx.x; i + 32768 < len; i += RESOLVE_THREADS)
    bad |= !resolve_value(arena[off + i], off, out, out[off + i]);
  if (bad) atomicExch(err, ERR_WINDOW);
}

}  // namespace

void launch_inflate_find(const uint8_t *in, uint64_t n, uint64_t span, uint32_t n_spans, uint64_t *cand, cudaStream_t s) {
  if (n_spans < 2) return;
  const uint32_t smem = FIND_THREADS * sizeof(HdrScratch);
  cudaFuncSetAttribute(lb2_inflate_find_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  lb2_inflate_find_kernel<<<(n_spans - 1 + FIND_THREADS / 32 - 1) / (FIND_THREADS / 32), FIND_THREADS, smem, s>>>(in, n, span, n_spans, cand);
}
void launch_inflate_count(const uint8_t *in, uint64_t n, const SpanJob *jobs, uint32_t n_jobs, SpanResult *res, cudaStream_t s) {
  const uint32_t smem = SPAN_THREADS * sizeof(DecodeState);
  cudaFuncSetAttribute(lb2_inflate_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  lb2_inflate_count_kernel<<<(n_jobs + SPAN_THREADS - 1) / SPAN_THREADS, SPAN_THREADS, smem, s>>>(in, n, jobs, n_jobs, res);
}
void launch_inflate_decode(const uint8_t *in, uint64_t n, const SpanJob *jobs, uint32_t n_jobs, uint16_t *arena, int32_t *err,
                           cudaStream_t s) {
  const uint32_t smem = SPAN_THREADS * sizeof(DecodeState);
  cudaFuncSetAttribute(lb2_inflate_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  lb2_inflate_decode_kernel<<<(n_jobs + SPAN_THREADS - 1) / SPAN_THREADS, SPAN_THREADS, smem, s>>>(in, n, jobs, n_jobs, arena, err);
}
void launch_inflate_resolve(const uint16_t *arena, uint8_t *out, const SpanJob *jobs, uint32_t n_jobs, int32_t *err, cudaStream_t s) {
  lb2_inflate_window_kernel<<<1, WINDOW_THREADS, 0, s>>>(arena, out, jobs, n_jobs, err);
  lb2_inflate_resolve_kernel<<<n_jobs, RESOLVE_THREADS, 0, s>>>(arena, out, jobs, err);
}

}  // namespace lb2
