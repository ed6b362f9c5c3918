// elf_deps.cuh -- what the dynamic loader reads of a shared object before it maps it, behind lb2_elf_deps (kernels in
// elf_deps.cu), shared with the CPU emulator of the tests (tests/emu/deps_emu.cpp).
//
// Of an ELF64 little-endian object it reads the header (class, data, e_type, e_machine, e_phoff, e_phnum), the program
// headers (PT_DYNAMIC and the PT_LOADs), the dynamic array up to DT_NULL or the segment's end, the strings of
// DT_SONAME / DT_NEEDED / DT_RPATH / DT_RUNPATH, the version-needs chain (DT_VERNEED: each vn_file and its vna_names
// with their flags) and the version-definitions chain (DT_VERDEF: the first vda_name of each Verdef).  Addresses are
// mapped to file offsets through the first PT_LOAD whose file image holds them, as readelf's offset_from_vma does.
//
// Records come out in this order: the string tags in dynamic-array order (so DT_NEEDED keeps the order the loader's
// breadth-first search depends on), then the version needs (a VERNEED_FILE record, then one VERNEED_VERSION record
// per Vernaux naming that file record), then the version definitions.  Where several entries carry one of the scalar
// tags (DT_STRTAB, DT_STRSZ, DT_VER*), the last wins, as in glibc's get_dynamic_info and in readelf.
//
// Bounds: no byte outside [0, n) is read, whatever the bytes are.  Every offset is checked against n before it is
// read; every address must map into a PT_LOAD's file image, and what is read from there must stay inside that image;
// strings must end (NUL) before DT_STRSZ and the image's end; the version chains are walked at most their declared
// count, each link checked, and all of them together at most n / 8 + 2 entries (every entry takes 8 bytes or more),
// so a cyclic or overlapping chain ends.  Any of these failing makes the object ST_MALFORMED.
//
// The scans run through a Lanes object: for the kernel one warp, whose 32 lanes test 32 program headers, dynamic
// entries or string bytes at a time and find the first (or last) hit with a ballot; for the emulator one thread.
// Every lane runs the same parse on the same values, so the control flow stays uniform.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define ED_HD __host__ __device__ __forceinline__
#else
#define ED_HD inline
#endif

namespace lb2 {
namespace elfd {

// per-object status (LB2_ELF_* in lambdipy_b200.h)
enum : int32_t { ST_OK = 0, ST_NOT_ELF = 1, ST_UNSUPPORTED = 2, ST_STATIC = 3, ST_MALFORMED = 4 };
// record kinds (LB2_ELF_REC_*)
enum : uint32_t { REC_SONAME = 1, REC_NEEDED = 2, REC_RPATH = 3, REC_RUNPATH = 4, REC_VERNEED_FILE = 5,
                  REC_VERNEED_VERSION = 6, REC_VERDEF = 7 };

constexpr uint32_t PT_LOAD = 1, PT_DYNAMIC = 2;
constexpr uint64_t DT_NULL = 0, DT_NEEDED = 1, DT_STRTAB = 5, DT_STRSZ = 10, DT_SONAME = 14, DT_RPATH = 15,
                   DT_RUNPATH = 29, DT_VERDEF = 0x6ffffffc, DT_VERDEFNUM = 0x6ffffffd, DT_VERNEED = 0x6ffffffe,
                   DT_VERNEEDNUM = 0x6fffffff;
constexpr uint64_t EHDR = 64, PHDR = 56, DYN = 16, VERNEED = 16, VERNAUX = 16, VERDEF = 20, VERDAUX = 8;

// one record: a string of the pool, pool[off .. off + len) followed by a NUL (lb2_elf_record)
struct Record {
  uint32_t kind;   // REC_*
  uint32_t flags;  // VERNEED_VERSION: vna_flags (VER_FLG_WEAK = 2); VERDEF: vd_flags (VER_FLG_BASE = 1); else 0
  uint32_t ref;    // VERNEED_VERSION: the index of its VERNEED_FILE record among the object's records; else 0
  uint32_t len;
  uint64_t off;
};

// per object (lb2_elf_object): the count pass fills status .. pool_len, the host scan first_record and pool_off
struct Object {
  int32_t status;
  uint16_t machine, type;  // e_machine, e_type (0 unless the header is ELF64 little-endian and complete)
  uint32_t first_record, n_records;
  uint64_t pool_off, pool_len;
};

ED_HD uint64_t rd(const uint8_t *p, uint64_t off, int bytes) {  // little-endian, any alignment
  uint64_t v = 0;
  for (int i = bytes - 1; i >= 0; i--) v = v << 8 | p[off + i];
  return v;
}

// [off, off + len) inside [0, end): without overflow
ED_HD bool inside(uint64_t off, uint64_t len, uint64_t end) { return off <= end && len <= end - off; }

// The one-thread Lanes: the emulator's, and the reference the warp's must agree with.
struct SerialLanes {
  template <class P> uint64_t first(uint64_t from, uint64_t to, P pred) {
    for (uint64_t i = from; i < to; i++)
      if (pred(i)) return i;
    return to;
  }
  template <class P> uint64_t last(uint64_t from, uint64_t to, P pred) {  // `to` when none
    for (uint64_t i = to; i > from; i--)
      if (pred(i - 1)) return i - 1;
    return to;
  }
  bool leader() const { return true; }
  void copy(uint8_t *dst, const uint8_t *src, uint64_t len) {
    for (uint64_t i = 0; i < len; i++) dst[i] = src[i];
  }
};

// Sinks: Count sizes an object's records and pool, Write lays them out where the scan put them.
struct Count {
  uint32_t n = 0;
  uint64_t pool = 0;
  template <class L> ED_HD uint32_t emit(L &, uint32_t, uint32_t, uint32_t, const uint8_t *, uint64_t len) {
    pool += len + 1;
    return n++;
  }
};

struct Write {
  Record *rec;     // the object's first record
  uint8_t *pool;   // the whole pool
  uint64_t base;   // the object's first pool byte
  uint32_t cap;    // records counted for the object: never written past, whatever the second parse does
  uint64_t pool_cap;
  uint32_t n = 0;
  uint64_t used = 0;
  template <class L> ED_HD uint32_t emit(L &lanes, uint32_t kind, uint32_t flags, uint32_t ref, const uint8_t *s, uint64_t len) {
    if (n < cap && inside(used, len + 1, pool_cap)) {
      if (lanes.leader()) {
        rec[n] = Record{kind, flags, ref, (uint32_t)len, base + used};
        pool[base + used + len] = 0;
      }
      lanes.copy(pool + base + used, s, len);
    }
    used += len + 1;
    return n++;
  }
};

struct Seg {
  uint64_t off, end;  // the file image of the PT_LOAD an address fell in: [off, end)
};

template <class L> struct Parser {
  L &lanes;
  const uint8_t *p;
  uint64_t n, phoff, phnum;

  ED_HD uint32_t ph_type(uint64_t i) const { return (uint32_t)rd(p, phoff + i * PHDR, 4); }
  ED_HD uint64_t ph(uint64_t i, uint64_t field) const { return rd(p, phoff + i * PHDR + field, 8); }

  // the file offset of the address a, with `len` bytes from there inside the same PT_LOAD's file image.  Address 0
  // is refused: there lies the ELF header, and readelf reads a table tag of 0 as absent.
  ED_HD bool map(uint64_t a, uint64_t len, uint64_t &off, Seg &seg) {
    if (a == 0) return false;
    const uint64_t i = lanes.first(0, phnum, [&](uint64_t k) {
      if (ph_type(k) != PT_LOAD) return false;
      const uint64_t va = ph(k, 16), fs = ph(k, 32);
      return a >= va && a - va < fs;
    });
    if (i == phnum) return false;
    const uint64_t va = ph(i, 16), po = ph(i, 8), fs = ph(i, 32);
    if (!inside(po, fs, n)) return false;
    seg = Seg{po, po + fs};
    off = po + (a - va);
    return inside(off, len, seg.end);
  }
};

// The parse: the object's status, its records handed to sink.emit in order.  machine / type receive e_machine and
// e_type once the header is known to be a complete ELF64 little-endian one.
template <class L, class S>
ED_HD int32_t parse(L &lanes, const uint8_t *p, uint64_t n, S &sink, uint16_t &machine, uint16_t &type) {
  machine = type = 0;
  if (n < 4 || p[0] != 0x7f || p[1] != 'E' || p[2] != 'L' || p[3] != 'F') return ST_NOT_ELF;
  if (n < 16) return ST_MALFORMED;
  const uint8_t cls = p[4], data = p[5];
  if (!(cls == 2 && data == 1)) return (cls == 1 || cls == 2) && (data == 1 || data == 2) ? ST_UNSUPPORTED : ST_MALFORMED;
  if (n < EHDR) return ST_MALFORMED;
  type = (uint16_t)rd(p, 16, 2);
  machine = (uint16_t)rd(p, 18, 2);
  Parser<L> ps{lanes, p, n, rd(p, 32, 8), rd(p, 56, 2)};
  if (ps.phnum == 0) return ST_STATIC;
  if (ps.phnum == 0xffff || rd(p, 54, 2) != PHDR || !inside(ps.phoff, ps.phnum * PHDR, n)) return ST_MALFORMED;
  const uint64_t di = lanes.first(0, ps.phnum, [&](uint64_t k) { return ps.ph_type(k) == PT_DYNAMIC; });
  if (di == ps.phnum) return ST_STATIC;
  const uint64_t d0 = ps.ph(di, 8), dsz = ps.ph(di, 32);
  if (!inside(d0, dsz, n)) return ST_MALFORMED;
  auto tag = [&](uint64_t k) { return rd(p, d0 + k * DYN, 8); };
  auto val = [&](uint64_t k) { return rd(p, d0 + k * DYN + 8, 8); };
  const uint64_t end = lanes.first(0, dsz / DYN, [&](uint64_t k) { return tag(k) == DT_NULL; });
  auto last = [&](uint64_t t) { return lanes.last(0, end, [&](uint64_t k) { return tag(k) == t; }); };
  auto is_str = [](uint64_t t) { return t == DT_NEEDED || t == DT_SONAME || t == DT_RPATH || t == DT_RUNPATH; };
  const uint64_t i_strtab = last(DT_STRTAB), i_strsz = last(DT_STRSZ), i_vn = last(DT_VERNEED),
                 i_vnnum = last(DT_VERNEEDNUM), i_vd = last(DT_VERDEF), i_vdnum = last(DT_VERDEFNUM);
  const bool any_str = lanes.first(0, end, [&](uint64_t k) { return is_str(tag(k)); }) < end;
  if (!(any_str || i_vn < end || i_vd < end)) return ST_OK;
  // the string table: mapped whole when its size is known, else from its start to its segment's end
  if (i_strtab == end) return ST_MALFORMED;
  uint64_t str0, str_end;
  Seg seg;
  if (i_strsz < end) {
    if (!ps.map(val(i_strtab), val(i_strsz), str0, seg)) return ST_MALFORMED;
    str_end = str0 + val(i_strsz);
  } else {
    if (!ps.map(val(i_strtab), 0, str0, seg) || str0 == seg.end) return ST_MALFORMED;
    str_end = seg.end;
  }
  // a string: offset v of the table, its length found by a vote for the NUL
  auto str = [&](uint64_t v, uint64_t &at, uint64_t &len) {
    if (v >= str_end - str0) return false;
    at = str0 + v;
    const uint64_t z = lanes.first(at, str_end, [&](uint64_t k) { return p[k] == 0; });
    len = z - at;
    return z < str_end && len < 0xffffffffu;
  };
  uint64_t at, len;
  for (uint64_t k = lanes.first(0, end, [&](uint64_t j) { return is_str(tag(j)); }); k < end;
       k = lanes.first(k + 1, end, [&](uint64_t j) { return is_str(tag(j)); })) {
    const uint64_t t = tag(k);
    if (!str(val(k), at, len)) return ST_MALFORMED;
    sink.emit(lanes, t == DT_NEEDED ? REC_NEEDED : t == DT_SONAME ? REC_SONAME : t == DT_RPATH ? REC_RPATH : REC_RUNPATH,
              0, 0, p + at, len);
  }
  uint64_t budget = n / 8 + 2;  // chain entries visited, all chains together
  if (i_vn < end) {
    if (i_vnnum == end) return ST_MALFORMED;
    const uint64_t num = val(i_vnnum);
    uint64_t off;
    if (!ps.map(val(i_vn), VERNEED, off, seg)) return ST_MALFORMED;
    for (uint64_t c = 0; c < num; c++) {
      if (!budget-- || !inside(off, VERNEED, seg.end)) return ST_MALFORMED;
      const uint64_t cnt = rd(p, off + 2, 2), aux = rd(p, off + 8, 4), next = rd(p, off + 12, 4);
      if (!str(rd(p, off + 4, 4), at, len)) return ST_MALFORMED;
      const uint32_t file = sink.emit(lanes, REC_VERNEED_FILE, 0, 0, p + at, len);
      uint64_t a = off + aux;
      for (uint64_t j = 0; j < cnt; j++) {
        if (!budget-- || !inside(a, VERNAUX, seg.end)) return ST_MALFORMED;
        if (!str(rd(p, a + 8, 4), at, len)) return ST_MALFORMED;
        sink.emit(lanes, REC_VERNEED_VERSION, (uint32_t)rd(p, a + 4, 2), file, p + at, len);
        const uint64_t an = rd(p, a + 12, 4);
        if (j + 1 < cnt && an == 0) return ST_MALFORMED;  // the chain ends before vn_cnt entries
        a += an;
      }
      if (c + 1 < num && next < VERNEED) return ST_MALFORMED;  // ends, or steps inside its own entry, before the count
      off += next;
    }
  }
  if (i_vd < end) {
    if (i_vdnum == end) return ST_MALFORMED;
    const uint64_t num = val(i_vdnum);
    uint64_t off;
    if (!ps.map(val(i_vd), VERDEF, off, seg)) return ST_MALFORMED;
    for (uint64_t c = 0; c < num; c++) {
      if (!budget-- || !inside(off, VERDEF, seg.end)) return ST_MALFORMED;
      const uint64_t flags = rd(p, off + 2, 2), cnt = rd(p, off + 6, 2), aux = rd(p, off + 12, 4), next = rd(p, off + 16, 4);
      if (cnt) {
        const uint64_t a = off + aux;
        if (!inside(a, VERDAUX, seg.end) || !str(rd(p, a, 4), at, len)) return ST_MALFORMED;
        sink.emit(lanes, REC_VERDEF, (uint32_t)flags, 0, p + at, len);
      }
      if (c + 1 < num && next < VERDEF) return ST_MALFORMED;
      off += next;
    }
  }
  return ST_OK;
}

}  // namespace elfd
}  // namespace lb2
