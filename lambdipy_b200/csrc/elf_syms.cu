// elf_syms.cu -- the symbol lookups of shared objects in device memory behind lb2_syms_* (api.cu); the logic itself is
// elf_syms.cuh.
//
// Index (one warp per object): a count pass sizes each object's tables, the host places them in the arena, a write
// pass copies them there and fills the version table.  References: a grid-stride pass over every object's relocation
// entries marks the referenced undefined symbols in each object's bitmap; a count pass (one warp per object) counts
// and checks them, the host places the Ref arrays, and a write pass compacts the bitmap into them.  Resolve: one warp
// per (reference, scope); the lanes look the symbol up in 32 objects of the scope at a time and a ballot keeps the
// first that defines it.  Find: one warp per query, the same 32-at-a-time probe of a name the host uploaded.
#include "lb2_common.cuh"
#include "elf_syms.cuh"

namespace lb2 {
using SymJob = elfs::Job;
using SymMiss = elfs::Miss;
using SymQuery = elfs::Query;
using SymFound = elfs::Found;
namespace {
using elfs::Object;
using elfs::Ref;

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
      const uint64_t i = e - 1 - lane;
      const uint32_t m = __ballot_sync(0xFFFFFFFFu, e - from > lane && pred(i));
      if (m) return e - 1 - (__ffs(m) - 1);
    }
    return to;
  }
  template <class F> __device__ uint64_t max(uint64_t from, uint64_t to, F f) {
    unsigned long long m = 0;
    for (uint64_t i = from + lane; i < to; i += 32) {
      const unsigned long long v = f(i);
      m = v > m ? v : m;
    }
    for (int d = 16; d; d >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xFFFFFFFFu, m, d);
      m = o > m ? o : m;
    }
    return m;
  }
  template <class P> __device__ bool any(uint64_t from, uint64_t to, P pred) {
    bool hit = false;
    for (uint64_t i = from + lane; i < to && !hit; i += 32) hit = pred(i);
    return __any_sync(0xFFFFFFFFu, hit);
  }
  __device__ bool leader() const { return lane == 0; }
  __device__ void copy(uint8_t *dst, const uint8_t *src, uint64_t len) {
    for (uint64_t i = lane; i < len; i += 32) dst[i] = src[i];
    __syncwarp();
  }
};

constexpr int WARPS = 4;

__global__ void __launch_bounds__(32 * WARPS) lb2_syms_index_count_kernel(const uint64_t *ptrs, const uint64_t *sizes,
                                                                          uint32_t n, Object *obj) {
  const uint32_t i = blockIdx.x * WARPS + threadIdx.x / 32;
  if (i >= n) return;
  WarpLanes lanes{threadIdx.x & 31};
  elfs::CountVer cv;
  Object o;
  const int32_t st = elfs::index(lanes, reinterpret_cast<const uint8_t *>(ptrs[i]), sizes[i], o, cv);
  if (lanes.leader()) {
    if (st != elfs::ST_OK) o = Object{};
    o.status = st;
    obj[i] = o;
  }
}

// the host has set obj[i].arena and zeroed the block: the tables copied, the version table filled
__global__ void __launch_bounds__(32 * WARPS) lb2_syms_index_write_kernel(const uint64_t *ptrs, const uint64_t *sizes,
                                                                          uint32_t n, const Object *obj) {
  const uint32_t i = blockIdx.x * WARPS + threadIdx.x / 32;
  if (i >= n || obj[i].status != elfs::ST_OK) return;
  WarpLanes lanes{threadIdx.x & 31};
  const Object o = obj[i];
  const uint8_t *p = reinterpret_cast<const uint8_t *>(ptrs[i]);
  uint8_t *a = reinterpret_cast<uint8_t *>(o.arena);
  const elfs::Tables t = elfs::tables(o);
  elfs::WriteVer wv{reinterpret_cast<elfs::Ver *>(a + t.ver), o.nver, lanes.leader()};
  Object again;
  elfs::index(lanes, p, sizes[i], again, wv);
  lanes.copy(a + t.sym, p + o.sym_off, (uint64_t)o.nsyms * elfs::SYM);
  if (o.flags & elfs::F_VERSYM) lanes.copy(a + t.versym, p + o.versym_off, 2ull * o.nsyms);
  lanes.copy(a + t.hash, p + o.hash_off, o.hash_len);
  lanes.copy(a + t.str, p + o.str_off, o.str_len);
}

// entry g of all objects' relocations: base[i] .. base[i + 1] are object i's
__global__ void lb2_syms_mark_kernel(const uint64_t *ptrs, const uint64_t *base, uint32_t n, Object *obj) {
  const uint64_t total = base[n];
  for (uint64_t g = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; g < total; g += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = n;  // the object: the last i with base[i] <= g
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) / 2;
      if (base[mid] <= g) lo = mid; else hi = mid;
    }
    const Object &o = obj[lo];
    if (o.status != elfs::ST_OK) continue;
    uint8_t *a = reinterpret_cast<uint8_t *>(o.arena);
    const int64_t s = elfs::mark(reinterpret_cast<const uint8_t *>(ptrs[lo]), o, a, g - base[lo]);
    if (s >= 0)
      atomicOr(reinterpret_cast<uint32_t *>(a + elfs::tables(o).bits) + s / 32, 1u << (s % 32));
    else if (s == -2)
      atomicOr(&obj[lo].flags, (uint32_t)elfs::F_BAD_REL);
  }
}

__global__ void __launch_bounds__(32 * WARPS) lb2_syms_refs_count_kernel(uint32_t n, Object *obj) {
  const uint32_t i = blockIdx.x * WARPS + threadIdx.x / 32;
  if (i >= n || obj[i].status != elfs::ST_OK) return;
  const uint32_t lane = threadIdx.x & 31;
  const Object o = obj[i];
  const uint8_t *a = reinterpret_cast<const uint8_t *>(o.arena);
  const uint32_t *bits = reinterpret_cast<const uint32_t *>(a + elfs::tables(o).bits);
  uint32_t cnt = 0;
  bool bad = false;
  for (uint32_t w = lane; w < (o.nsyms + 31) / 32; w += 32)
    for (uint32_t m = bits[w]; m; m &= m - 1) {
      Ref r;
      bad |= !elfs::make_ref(o, a, w * 32 + __ffs(m) - 1, r);
      cnt++;
    }
  cnt = __reduce_add_sync(0xFFFFFFFFu, cnt);
  bad = __any_sync(0xFFFFFFFFu, bad);
  if (lane == 0) {
    if (bad || (o.flags & elfs::F_BAD_REL)) {
      obj[i].status = elfs::ST_MALFORMED;
      obj[i].nrefs = 0;
    } else {
      obj[i].nrefs = cnt;
    }
  }
}

// the host has set obj[i].refs: the marked symbols in index order, 32 bitmap words per step, a warp scan of their
// counts placing each lane's
__global__ void __launch_bounds__(32 * WARPS) lb2_syms_refs_write_kernel(uint32_t n, const Object *obj) {
  const uint32_t i = blockIdx.x * WARPS + threadIdx.x / 32;
  if (i >= n || obj[i].status != elfs::ST_OK || !obj[i].nrefs) return;
  const uint32_t lane = threadIdx.x & 31;
  const Object o = obj[i];
  const uint8_t *a = reinterpret_cast<const uint8_t *>(o.arena);
  const uint32_t *bits = reinterpret_cast<const uint32_t *>(a + elfs::tables(o).bits);
  Ref *out = reinterpret_cast<Ref *>(o.refs);
  const uint32_t words = (o.nsyms + 31) / 32;
  uint32_t at = 0;
  for (uint32_t w0 = 0; w0 < words; w0 += 32) {
    const uint32_t w = w0 + lane, m0 = w < words ? bits[w] : 0, c = __popc(m0);
    uint32_t x = c;  // inclusive scan
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d);
      if (lane >= d) x += y;
    }
    uint32_t k = at + x - c;
    for (uint32_t m = m0; m; m &= m - 1, k++)
      if (k < o.nrefs) elfs::make_ref(o, a, w * 32 + __ffs(m) - 1, out[k]);
    at += __shfl_sync(0xFFFFFFFFu, x, 31);
  }
}

// One warp per (job, reference): jobs[j] resolves the references of objs[jobs[j].obj] in the scope
// scope[jobs[j].scope_off ..+ scope_len); ref_base[j] .. ref_base[j + 1] number its references globally.
__global__ void __launch_bounds__(32 * WARPS) lb2_syms_resolve_kernel(const Object *objs, const SymJob *jobs,
                                                                      const uint64_t *ref_base, uint32_t n_jobs,
                                                                      const uint32_t *scope, const uint8_t *cls,
                                                                      uint32_t *counts, SymMiss *miss, uint32_t max_miss,
                                                                      uint32_t *n_miss, unsigned long long *lookups) {
  const uint64_t total = ref_base[n_jobs], warps = (uint64_t)gridDim.x * WARPS;
  const uint32_t lane = threadIdx.x & 31;
  unsigned long long probed = 0;
  for (uint64_t g = blockIdx.x * (uint64_t)WARPS + threadIdx.x / 32; g < total; g += warps) {
    uint32_t lo = 0, hi = n_jobs;
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) / 2;
      if (ref_base[mid] <= g) lo = mid; else hi = mid;
    }
    const SymJob jb = jobs[lo];
    const Object &o = objs[jb.obj];
    const uint8_t *oa = reinterpret_cast<const uint8_t *>(o.arena);
    const uint32_t k = (uint32_t)(g - ref_base[lo]);
    const Ref r = reinterpret_cast<const Ref *>(o.refs)[k];
    const elfs::Ver *rv = elfs::ref_version(o, oa, r);
    int32_t found = -1;
    for (uint32_t b = 0; b < jb.scope_len && found < 0; b += 32) {
      bool hit = false;
      if (b + lane < jb.scope_len) {
        const Object &d = objs[scope[jb.scope_off + b + lane]];
        hit = elfs::lookup(d, reinterpret_cast<const uint8_t *>(d.arena), o, oa, r, rv) >= 0;
      }
      const uint32_t m = __ballot_sync(0xFFFFFFFFu, hit);
      if (m) found = (int32_t)(b + __ffs(m) - 1);
    }
    if (lane == 0) {
      probed += found >= 0 ? found + 1 : jb.scope_len;
      if (found >= 0)
        atomicAdd(&counts[3 * lo + cls[scope[jb.scope_off + found]]], 1u);
      else if (!r.weak) {
        const uint32_t at = atomicAdd(n_miss, 1u);
        if (at < max_miss) miss[at] = SymMiss{lo, k};
      }
    }
  }
  if (lane == 0 && probed) atomicAdd(lookups, probed);
}

// One warp per query: the name pool[name_off ..+ name_len) looked up as dlsym looks it up (newest) in scope[scope_off
// ..+ scope_len); every lane hashes the name, then probes one scope entry of each 32.  The host has checked that
// every query lies inside the pool and the scope array and that every scope entry is an object id.
__global__ void __launch_bounds__(32 * WARPS) lb2_syms_find_kernel(const Object *objs, const SymQuery *queries, uint32_t n,
                                                                   const uint32_t *scope, const uint8_t *pool,
                                                                   SymFound *found) {
  const uint32_t q = blockIdx.x * WARPS + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (q >= n) return;
  const SymQuery qy = queries[q];
  const uint8_t *name = pool + qy.name_off;
  const uint32_t gnu = elfs::gnu_hash(name, qy.name_len), sysv = elfs::sysv_hash(name, qy.name_len);
  int64_t sym = -1;
  uint32_t at = 0;
  for (uint32_t b = 0; b < qy.scope_len; b += 32) {
    int64_t s = -1;
    if (b + lane < qy.scope_len) {
      const Object &d = objs[scope[qy.scope_off + b + lane]];
      s = elfs::lookup_name(d, reinterpret_cast<const uint8_t *>(d.arena), name, qy.name_len, gnu, sysv, nullptr,
                            nullptr, true);
    }
    const uint32_t m = __ballot_sync(0xFFFFFFFFu, s >= 0);
    if (m) {
      const int first = __ffs(m) - 1;
      at = b + first;
      sym = __shfl_sync(0xFFFFFFFFu, s, first);
      break;
    }
  }
  if (lane == 0) {
    if (sym < 0) {
      found[q] = SymFound{elfs::NOT_FOUND, 0, 0, 0, 0};
    } else {
      const uint32_t id = scope[qy.scope_off + at];
      found[q] = elfs::found_at(id, objs[id], reinterpret_cast<const uint8_t *>(objs[id].arena), (uint32_t)sym);
    }
  }
}

// the strings of a missed reference: name, version name, version file, each followed by a NUL
__device__ void miss_strings(const Object *objs, const SymJob *jobs, const SymMiss &m, const uint8_t *s[3], uint32_t len[3]) {
  const Object &o = objs[jobs[m.job].obj];
  const uint8_t *a = reinterpret_cast<const uint8_t *>(o.arena), *str = a + elfs::tables(o).str;
  const Ref r = reinterpret_cast<const Ref *>(o.refs)[m.ref];
  const elfs::Ver *v = elfs::ref_version(o, a, r);
  s[0] = str + r.name, len[0] = r.name_len;
  s[1] = v ? str + v->name : str, len[1] = v ? v->name_len : 0;
  s[2] = v && v->file != elfs::NO_STR ? str + v->file : str, len[2] = v && v->file != elfs::NO_STR ? v->file_len : 0;
}

__global__ void lb2_syms_names_count_kernel(const Object *objs, const SymJob *jobs, const SymMiss *miss, uint32_t n,
                                            uint64_t *len) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t *s[3];
  uint32_t l[3];
  miss_strings(objs, jobs, miss[i], s, l);
  len[i] = (uint64_t)l[0] + l[1] + l[2] + 3;
}

__global__ void lb2_syms_names_write_kernel(const Object *objs, const SymJob *jobs, const SymMiss *miss, uint32_t n,
                                            const uint64_t *off, uint8_t *pool) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t *s[3];
  uint32_t l[3];
  miss_strings(objs, jobs, miss[i], s, l);
  uint8_t *d = pool + off[i];
  for (int k = 0; k < 3; k++) {
    for (uint32_t j = 0; j < l[k]; j++) *d++ = s[k][j];
    *d++ = 0;
  }
}

}  // namespace

void launch_syms_index_count(const uint64_t *ptrs, const uint64_t *sizes, uint32_t n, void *obj, cudaStream_t s) {
  if (n) lb2_syms_index_count_kernel<<<(n + WARPS - 1) / WARPS, 32 * WARPS, 0, s>>>(ptrs, sizes, n, static_cast<Object *>(obj));
}

void launch_syms_index_write(const uint64_t *ptrs, const uint64_t *sizes, uint32_t n, const void *obj, cudaStream_t s) {
  if (n) lb2_syms_index_write_kernel<<<(n + WARPS - 1) / WARPS, 32 * WARPS, 0, s>>>(ptrs, sizes, n, static_cast<const Object *>(obj));
}

void launch_syms_refs(const uint64_t *ptrs, const uint64_t *rel_base, uint64_t total_rel, uint32_t n, void *obj,
                      cudaStream_t s) {
  if (!n) return;
  if (total_rel) {
    const uint64_t blocks = (total_rel + 255) / 256;
    lb2_syms_mark_kernel<<<(unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, s>>>(ptrs, rel_base, n, static_cast<Object *>(obj));
  }
  lb2_syms_refs_count_kernel<<<(n + WARPS - 1) / WARPS, 32 * WARPS, 0, s>>>(n, static_cast<Object *>(obj));
}

void launch_syms_refs_write(uint32_t n, const void *obj, cudaStream_t s) {
  if (n) lb2_syms_refs_write_kernel<<<(n + WARPS - 1) / WARPS, 32 * WARPS, 0, s>>>(n, static_cast<const Object *>(obj));
}

void launch_syms_resolve(const void *objs, const SymJob *jobs, const uint64_t *ref_base, uint32_t n_jobs, uint64_t total,
                         const uint32_t *scope, const uint8_t *cls, uint32_t *counts, SymMiss *miss, uint32_t max_miss,
                         uint32_t *n_miss, unsigned long long *lookups, cudaStream_t s) {
  if (!n_jobs || !total) return;
  const uint64_t blocks = (total + WARPS - 1) / WARPS;
  lb2_syms_resolve_kernel<<<(unsigned)(blocks < 65536 ? blocks : 65536), 32 * WARPS, 0, s>>>(
      static_cast<const Object *>(objs), jobs, ref_base, n_jobs, scope, cls, counts, miss, max_miss, n_miss, lookups);
}

void launch_syms_names(const void *objs, const SymJob *jobs, const SymMiss *miss, uint32_t n, uint64_t *len_or_off,
                       uint8_t *pool, cudaStream_t s) {
  if (!n) return;
  if (!pool)
    lb2_syms_names_count_kernel<<<(n + 127) / 128, 128, 0, s>>>(static_cast<const Object *>(objs), jobs, miss, n, len_or_off);
  else
    lb2_syms_names_write_kernel<<<(n + 127) / 128, 128, 0, s>>>(static_cast<const Object *>(objs), jobs, miss, n, len_or_off, pool);
}

void launch_syms_find(const void *objs, const SymQuery *queries, uint32_t n, const uint32_t *scope, const uint8_t *pool,
                      SymFound *found, cudaStream_t s) {
  if (n) lb2_syms_find_kernel<<<(n + WARPS - 1) / WARPS, 32 * WARPS, 0, s>>>(static_cast<const Object *>(objs), queries, n,
                                                                             scope, pool, found);
}

}  // namespace lb2
