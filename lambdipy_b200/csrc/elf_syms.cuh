// elf_syms.cuh -- the symbol lookups the dynamic loader does when it relocates a shared object, behind lb2_syms_*
// (kernels in elf_syms.cu), shared with the CPU emulator of the tests (tests/emu/syms_emu.cpp).  The rules restate
// glibc's elf/dl-lookup.c (do_lookup_x, check_match), elf/dl-version.c (_dl_check_map_versions: the l_versions
// table) and elf/do-rel.h with elf/dl-reloc.c (RESOLVE_MAP: which relocations look a symbol up, with which version).
//
// Three steps, each a function here:
//  * index: of an object that lies in device memory, the tables a lookup needs -- .dynsym (DT_SYMTAB), .dynstr,
//    .gnu.version (DT_VERSYM), the hash table (DT_GNU_HASH, else DT_HASH) -- and its version table, indexed by versym
//    index as glibc's l_versions: {hash, name, file, hidden} of each non-base Verdef (vd_ndx) and each Vernaux
//    (vna_other).  The tables are copied into a persistent arena (tables()), because the object itself is gone once
//    the zip reader decodes its next batch.  The hashed symbols are DT_HASH's nchain, or up to the end of the GNU hash
//    chains; the copy also takes any symbol past them that a relocation names.
//  * references: every DT_RELA / DT_JMPREL entry with a symbol index > 0 whose symbol is SHN_UNDEF and not STB_LOCAL
//    marks that symbol in a per-object bitmap (mark()); the marked symbols, compacted in index order, are the
//    object's references, each with its GNU and SysV hash and its versym index.
//  * lookup: one reference in one object: bloom filter, bucket, chain, name compare and check_match.  A warp takes
//    32 objects of a scope at a time and a ballot keeps the first one in scope order that defines the symbol.
//  * find: the same lookup of a name given by the host, as dlsym(handle, name) does it (elf/dl-sym.c: the handle's
//    local scope, DL_LOOKUP_RETURN_NEWEST), for the PyInit_* export of a Python extension module.
//
// Bounds are elf_deps.cuh's: no byte outside [0, n) of an object is read; every table must map into a PT_LOAD's file
// image and fit there; strings must end before DT_STRSZ; version chains are walked at most their count and n / 8 + 2
// entries in all; a GNU hash chain end is searched only inside its segment, and chain walks in lookups are capped at
// the symbol count the hash table gives.  Lookups read only the arena copies, whose sizes the index fixed.
#pragma once
#include "elf_deps.cuh"

namespace lb2 {
namespace elfs {
using elfd::inside;
using elfd::rd;

// per-object status (LB2_SYM_*): the elf_deps statuses, of which OK, UNSUPPORTED and MALFORMED also say whether the
// symbol tables could be read
enum : int32_t { ST_OK = 0, ST_NOT_ELF = 1, ST_UNSUPPORTED = 2, ST_STATIC = 3, ST_MALFORMED = 4 };
// Object.flags (LB2_SYM_F_*)
enum : uint32_t { F_GNU = 1, F_SYSV = 2, F_VERSYM = 4, F_BAD_REL = 8 };

constexpr uint64_t DT_PLTRELSZ = 2, DT_HASH = 4, DT_SYMTAB = 6, DT_RELA = 7, DT_RELASZ = 8, DT_RELAENT = 9,
                   DT_SYMENT = 11, DT_REL = 17, DT_PLTREL = 20, DT_JMPREL = 23, DT_GNU_HASH = 0x6ffffef5,
                   DT_VERSYM = 0x6ffffff0;
constexpr uint64_t SYM = 24, RELA = 24, NO_STR = 0xffffffffu;
constexpr uint32_t SHN_UNDEF = 0, SHN_ABS = 0xfff1, STB_LOCAL = 0, STB_GLOBAL = 1, STB_WEAK = 2, STB_GNU_UNIQUE = 10,
                   STT_TLS = 6, VER_FLG_BASE = 1;
// dl-lookup.c ALLOWED_STT: NOTYPE, OBJECT, FUNC, COMMON, TLS, GNU_IFUNC
constexpr uint32_t ALLOWED_STT = (1u << 0) | (1u << 1) | (1u << 2) | (1u << 5) | (1u << 6) | (1u << 10);

// per object (lb2_sym_object).  The index fills everything but arena / refs (device addresses the host assigns) and
// nrefs (the reference count pass).
struct Object {
  int32_t status;
  uint32_t flags;                    // F_*
  uint32_t nsyms, nver;              // symbols copied, version-table entries (the highest versym index defined + 1)
  uint32_t nbucket, symoffset;       // GNU: nbuckets, symoffset; SysV: nbucket, 0
  uint32_t bloom_words, bloom_shift; // GNU only
  uint32_t nrefs, nhash;             // references; symbols the hash table covers (nsyms may be more)
  uint64_t str_len, hash_len;        // bytes of .dynstr and of the hash table
  uint64_t sym_off, str_off, versym_off, hash_off;  // file offsets of the tables
  uint64_t rela_off, rela_n, plt_off, plt_n;        // file offsets and entry counts of DT_RELA and DT_JMPREL
  uint64_t arena, refs;              // device addresses of the object's tables and of its Ref array
};

// one version-table entry (l_versions[i]); flags 1: set, 2: hidden (vna_other & 0x8000).  Strings are .dynstr offsets.
struct Ver {
  uint32_t hash, name, name_len, file, file_len, flags;
};

// one reference: a relocated undefined symbol
struct Ref {
  uint32_t sym;           // its .dynsym index
  uint32_t name, name_len;
  uint32_t gnu, sysv;     // dl_new_hash and _dl_elf_hash of its name
  uint16_t ver;           // versym index & 0x7fff, 0 without DT_VERSYM
  uint8_t weak, pad;
};

// resolve: the references of objects[obj] looked up in scope[scope_off ..+ scope_len) (lb2_sym_job); a strong reference
// found nowhere is reported as {job, ref} (lb2_sym_miss)
struct Job {
  uint32_t obj, scope_off, scope_len, pad;
};
struct Miss {
  uint32_t job, ref;
};

// where each table lies in the object's arena block (8-byte aligned pieces; .dynstr last, followed by one NUL)
struct Tables {
  uint64_t sym, versym, hash, ver, bits, str, end;
};
ED_HD uint64_t al8(uint64_t x) { return (x + 7) & ~7ull; }
ED_HD Tables tables(const Object &o) {
  Tables t;
  t.sym = 0;
  t.versym = al8(t.sym + (uint64_t)o.nsyms * SYM);
  t.hash = al8(t.versym + (o.flags & F_VERSYM ? (uint64_t)o.nsyms * 2 : 0));
  t.ver = al8(t.hash + o.hash_len);
  t.bits = al8(t.ver + (uint64_t)o.nver * sizeof(Ver));
  t.str = al8(t.bits + ((uint64_t)o.nsyms + 31) / 32 * 4);
  t.end = al8(t.str + o.str_len + 1);
  return t;
}

ED_HD uint32_t gnu_hash(const uint8_t *s, uint64_t len) {  // dl_new_hash
  uint32_t h = 5381;
  for (uint64_t i = 0; i < len; i++) h = h * 33 + s[i];
  return h;
}
ED_HD uint32_t sysv_hash(const uint8_t *s, uint64_t len) {  // _dl_elf_hash
  uint32_t h = 0;
  for (uint64_t i = 0; i < len; i++) {
    h = (h << 4) + s[i];
    const uint32_t g = h & 0xf0000000u;
    h ^= g >> 24;
    h &= ~g;
  }
  return h;
}

// elf_deps' SerialLanes with the reductions the index needs
struct SerialLanes : elfd::SerialLanes {
  template <class F> uint64_t max(uint64_t from, uint64_t to, F f) {  // max of f over [from, to), 0 when empty
    uint64_t m = 0;
    for (uint64_t i = from; i < to; i++) {
      const uint64_t v = f(i);
      m = v > m ? v : m;
    }
    return m;
  }
  template <class P> uint64_t any(uint64_t from, uint64_t to, P pred) { return first(from, to, pred) < to; }
};

struct NullSink {  // elf_deps' parse run for its status only
  template <class L> ED_HD uint32_t emit(L &, uint32_t, uint32_t, uint32_t, const uint8_t *, uint64_t) { return 0; }
};

// The version sinks: CountVer finds the table's size, WriteVer fills it (zeroed beforehand).
struct CountVer {
  uint32_t top = 0;
  bool any = false;
  ED_HD void put(uint32_t ndx, uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, bool) {
    top = ndx > top ? ndx : top;
    any = true;
  }
};
struct WriteVer {
  Ver *ver;
  uint32_t nver;
  bool leader;
  ED_HD void put(uint32_t ndx, uint32_t hash, uint32_t name, uint32_t name_len, uint32_t file, uint32_t file_len, bool hidden) {
    if (leader && ndx < nver) ver[ndx] = Ver{hash, name, name_len, file, file_len, 1u | (hidden ? 2u : 0u)};
  }
};

// The index of the object p[0, n): its status and o's fields (not arena / refs / nrefs); its version-table entries to
// vs.put(index, hash, name, name_len, file, file_len, hidden), in chain order (a later entry of the same index wins,
// as in dl-version.c).
template <class L, class V> ED_HD int32_t index(L &lanes, const uint8_t *p, uint64_t n, Object &o, V &vs) {
  o = Object{};
  {
    NullSink ns;
    uint16_t machine, type;
    const int32_t st = elfd::parse(lanes, p, n, ns, machine, type);
    if (st != elfd::ST_OK) return st;
  }
  // elfd::parse has checked the header, the program headers and the dynamic array's bounds
  elfd::Parser<L> ps{lanes, p, n, rd(p, 32, 8), rd(p, 56, 2)};
  const uint64_t di = lanes.first(0, ps.phnum, [&](uint64_t k) { return ps.ph_type(k) == elfd::PT_DYNAMIC; });
  const uint64_t d0 = ps.ph(di, 8), dsz = ps.ph(di, 32);
  auto tag = [&](uint64_t k) { return rd(p, d0 + k * elfd::DYN, 8); };
  auto val = [&](uint64_t k) { return rd(p, d0 + k * elfd::DYN + 8, 8); };
  const uint64_t end = lanes.first(0, dsz / elfd::DYN, [&](uint64_t k) { return tag(k) == elfd::DT_NULL; });
  auto last = [&](uint64_t t) { return lanes.last(0, end, [&](uint64_t k) { return tag(k) == t; }); };
  const uint64_t i_sym = last(DT_SYMTAB), i_str = last(elfd::DT_STRTAB), i_strsz = last(elfd::DT_STRSZ),
                 i_syment = last(DT_SYMENT), i_gnu = last(DT_GNU_HASH), i_hash = last(DT_HASH), i_versym = last(DT_VERSYM),
                 i_rela = last(DT_RELA), i_relasz = last(DT_RELASZ), i_relaent = last(DT_RELAENT),
                 i_jmprel = last(DT_JMPREL), i_pltrelsz = last(DT_PLTRELSZ), i_pltrel = last(DT_PLTREL),
                 i_rel = last(DT_REL), i_vn = last(elfd::DT_VERNEED), i_vnnum = last(elfd::DT_VERNEEDNUM),
                 i_vd = last(elfd::DT_VERDEF), i_vdnum = last(elfd::DT_VERDEFNUM);
  // DT_REL relocations (not x86_64 / aarch64): not guessed
  if (i_rel < end || (i_jmprel < end && i_pltrel < end && val(i_pltrel) == DT_REL)) return ST_UNSUPPORTED;
  if (i_syment < end && val(i_syment) != SYM) return ST_MALFORMED;
  elfd::Seg seg;
  uint64_t off;
  // .dynstr, as elf_deps maps it
  if (i_str < end) {
    if (i_strsz < end) {
      if (!ps.map(val(i_str), val(i_strsz), off, seg)) return ST_MALFORMED;
      o.str_len = val(i_strsz);
    } else {
      if (!ps.map(val(i_str), 0, off, seg) || off == seg.end) return ST_MALFORMED;
      o.str_len = seg.end - off;
    }
    o.str_off = off;
  }
  if (o.str_len >= NO_STR) return ST_MALFORMED;
  // a string of .dynstr: its length, false unless it ends inside the table
  auto str = [&](uint64_t v, uint32_t &len) {
    if (v >= o.str_len) return false;
    const uint64_t at = o.str_off + v, z = lanes.first(at, o.str_off + o.str_len, [&](uint64_t k) { return p[k] == 0; });
    len = (uint32_t)(z - at);
    return z < o.str_off + o.str_len;
  };
  // the hash table, and with it the symbol count
  if (i_gnu < end) {
    uint64_t h0;
    if (!ps.map(val(i_gnu), 16, h0, seg)) return ST_MALFORMED;
    o.flags |= F_GNU;
    o.nbucket = (uint32_t)rd(p, h0, 4);
    o.symoffset = (uint32_t)rd(p, h0 + 4, 4);
    o.bloom_words = (uint32_t)rd(p, h0 + 8, 4);
    o.bloom_shift = (uint32_t)rd(p, h0 + 12, 4);
    if (!o.bloom_words || (o.bloom_words & (o.bloom_words - 1)) || o.bloom_shift >= 32) return ST_MALFORMED;
    const uint64_t b0 = h0 + 16 + 8ull * o.bloom_words, c0 = b0 + 4ull * o.nbucket;
    if (!inside(b0, 4ull * o.nbucket, seg.end)) return ST_MALFORMED;
    // a bucket names the first symbol of its chain, at symoffset or above
    if (lanes.any(0, o.nbucket, [&](uint64_t k) { const uint64_t b = rd(p, b0 + 4 * k, 4); return b && b < o.symoffset; }))
      return ST_MALFORMED;
    const uint64_t top = lanes.max(0, o.nbucket, [&](uint64_t k) { return rd(p, b0 + 4 * k, 4); });
    uint64_t nsyms = o.symoffset;
    if (top) {  // the last chain ends at the first word with bit 0 set from its start on
      const uint64_t words = (seg.end - c0) / 4;
      const uint64_t k = lanes.first(top - o.symoffset, words, [&](uint64_t j) { return rd(p, c0 + 4 * j, 4) & 1; });
      if (k == words) return ST_MALFORMED;
      nsyms = o.symoffset + k + 1;
    }
    if (nsyms >= 0xffffffffu) return ST_MALFORMED;
    o.nhash = (uint32_t)nsyms;
    o.hash_off = h0;
    o.hash_len = c0 - h0 + 4 * (nsyms - o.symoffset);
  } else if (i_hash < end) {
    uint64_t h0;
    if (!ps.map(val(i_hash), 8, h0, seg)) return ST_MALFORMED;
    o.flags |= F_SYSV;
    o.nbucket = (uint32_t)rd(p, h0, 4);
    o.nhash = (uint32_t)rd(p, h0 + 4, 4);
    o.hash_off = h0;
    o.hash_len = 8 + 4ull * o.nbucket + 4ull * o.nhash;
    if (!inside(h0, o.hash_len, seg.end)) return ST_MALFORMED;
  }
  // relocations with an addend: the whole DT_RELA table, and DT_JMPREL when DT_PLTREL says DT_RELA
  if (i_rela < end) {
    if ((i_relaent < end && val(i_relaent) != RELA) || i_relasz == end || val(i_relasz) % RELA) return ST_MALFORMED;
    if (val(i_relasz)) {
      if (!ps.map(val(i_rela), val(i_relasz), off, seg)) return ST_MALFORMED;
      o.rela_off = off;
      o.rela_n = val(i_relasz) / RELA;
    }
  }
  if (i_jmprel < end) {
    if (i_pltrel == end || val(i_pltrel) != DT_RELA || i_pltrelsz == end || val(i_pltrelsz) % RELA) return ST_MALFORMED;
    if (val(i_pltrelsz)) {
      if (!ps.map(val(i_jmprel), val(i_pltrelsz), off, seg)) return ST_MALFORMED;
      o.plt_off = off;
      o.plt_n = val(i_pltrelsz) / RELA;
    }
  }
  // the symbols: those the hash table covers, and any a relocation names past them (an executable's GNU hash table
  // leaves its undefined symbols out)
  {
    const uint64_t top = lanes.max(0, o.rela_n + o.plt_n, [&](uint64_t k) {
      return rd(p, (k < o.rela_n ? o.rela_off + k * RELA : o.plt_off + (k - o.rela_n) * RELA) + 8, 8) >> 32;
    });
    if (top >= 0xffffffffu) return ST_MALFORMED;
    o.nsyms = top + 1 > o.nhash ? (uint32_t)top + 1 : o.nhash;
    if (!top && !o.nhash) o.nsyms = 0;
  }
  if (o.nsyms) {
    if (i_sym == end || !ps.map(val(i_sym), (uint64_t)o.nsyms * SYM, off, seg)) return ST_MALFORMED;
    o.sym_off = off;
    if (!o.str_len) return ST_MALFORMED;
  }
  if (i_versym < end) {
    o.flags |= F_VERSYM;
    if (o.nsyms) {
      if (!ps.map(val(i_versym), 2ull * o.nsyms, off, seg)) return ST_MALFORMED;
      o.versym_off = off;
    }
  }
  // the version table, from the same chains elf_deps walks
  uint64_t budget = n / 8 + 2;
  uint32_t top = 0;
  bool any = false;
  auto put = [&](uint32_t ndx, uint32_t hash, uint64_t name, uint64_t file, bool hidden) {
    uint32_t nl = 0, fl = 0;
    if (!str(name, nl) || (file != NO_STR && !str(file, fl))) return false;
    vs.put(ndx, hash, (uint32_t)name, nl, (uint32_t)file, fl, hidden);
    top = ndx > top ? ndx : top;
    any = true;
    return true;
  };
  if (i_vn < end) {
    if (i_vnnum == end || !ps.map(val(i_vn), elfd::VERNEED, off, seg)) return ST_MALFORMED;
    const uint64_t num = val(i_vnnum);
    for (uint64_t c = 0; c < num; c++) {
      if (!budget-- || !inside(off, elfd::VERNEED, seg.end)) return ST_MALFORMED;
      const uint64_t cnt = rd(p, off + 2, 2), file = rd(p, off + 4, 4), next = rd(p, off + 12, 4);
      uint64_t a = off + rd(p, off + 8, 4);
      for (uint64_t j = 0; j < cnt; j++) {
        if (!budget-- || !inside(a, elfd::VERNAUX, seg.end)) return ST_MALFORMED;
        const uint32_t other = (uint32_t)rd(p, a + 6, 2);
        if (!put(other & 0x7fff, (uint32_t)rd(p, a, 4), rd(p, a + 8, 4), file, other & 0x8000)) return ST_MALFORMED;
        const uint64_t an = rd(p, a + 12, 4);
        if (j + 1 < cnt && an == 0) return ST_MALFORMED;
        a += an;
      }
      if (c + 1 < num && next < elfd::VERNEED) return ST_MALFORMED;
      off += next;
    }
  }
  if (i_vd < end) {
    if (i_vdnum == end || !ps.map(val(i_vd), elfd::VERDEF, off, seg)) return ST_MALFORMED;
    const uint64_t num = val(i_vdnum);
    for (uint64_t c = 0; c < num; c++) {
      if (!budget-- || !inside(off, elfd::VERDEF, seg.end)) return ST_MALFORMED;
      const uint64_t flags = rd(p, off + 2, 2), ndx = rd(p, off + 4, 2), cnt = rd(p, off + 6, 2), next = rd(p, off + 16, 4);
      if (cnt && !(flags & VER_FLG_BASE)) {  // the base version is not available for matching (dl-version.c)
        const uint64_t a = off + rd(p, off + 12, 4);
        if (!inside(a, elfd::VERDAUX, seg.end)) return ST_MALFORMED;
        if (!put((uint32_t)ndx & 0x7fff, (uint32_t)rd(p, off + 8, 4), rd(p, a, 4), NO_STR, false)) return ST_MALFORMED;
      }
      if (c + 1 < num && next < elfd::VERDEF) return ST_MALFORMED;
      off += next;
    }
  }
  o.nver = any ? top + 1 : 0;
  return ST_OK;
}

// Relocation entry k of the object (k < rela_n + plt_n): the symbol it names when that symbol is a reference, else
// -1; -2 when the index is past the symbol count (the object is then malformed).  sym: the arena's .dynsym copy.
ED_HD int64_t mark(const uint8_t *p, const Object &o, const uint8_t *sym, uint64_t k) {
  const uint64_t at = k < o.rela_n ? o.rela_off + k * RELA : o.plt_off + (k - o.rela_n) * RELA;
  const uint64_t s = rd(p, at + 8, 8) >> 32;  // ELF64_R_SYM(r_info)
  if (s == 0) return -1;
  if (s >= o.nsyms) return -2;
  const uint8_t info = sym[s * SYM + 4];
  return rd(sym, s * SYM + 6, 2) == SHN_UNDEF && (info >> 4) != STB_LOCAL ? (int64_t)s : -1;
}

// A reference's fields from the arena copies.  False when its name does not end inside .dynstr.
ED_HD bool make_ref(const Object &o, const uint8_t *a, uint32_t s, Ref &r) {
  const Tables t = tables(o);
  const uint64_t name = rd(a + t.sym, (uint64_t)s * SYM, 4);
  if (name >= o.str_len) return false;
  const uint8_t *str = a + t.str;
  uint64_t len = 0;
  while (name + len < o.str_len && str[name + len]) len++;
  if (name + len == o.str_len) return false;
  r.sym = s;
  r.name = (uint32_t)name;
  r.name_len = (uint32_t)len;
  r.gnu = gnu_hash(str + name, len);
  r.sysv = sysv_hash(str + name, len);
  r.ver = o.flags & F_VERSYM ? (uint16_t)(rd(a + t.versym, 2ull * s, 2) & 0x7fff) : 0;
  r.weak = (a[t.sym + (uint64_t)s * SYM + 4] >> 4) == STB_WEAK;
  r.pad = 0;
  return true;
}

// The version a reference asks for (RESOLVE_MAP: l_versions[ndx] when its hash is not 0), or null.
ED_HD const Ver *ref_version(const Object &o, const uint8_t *a, const Ref &r) {
  if (!(o.flags & F_VERSYM) || r.ver >= o.nver) return nullptr;
  const Ver *v = reinterpret_cast<const Ver *>(a + tables(o).ver) + r.ver;
  return (v->flags & 1) && v->hash ? v : nullptr;
}

ED_HD bool same(const uint8_t *x, const uint8_t *y, uint64_t len) {
  for (uint64_t i = 0; i < len; i++)
    if (x[i] != y[i]) return false;
  return true;
}

// do_lookup_x for one object: the index of the symbol of d (arena block da) named name[0, len) (gnu / sysv: its
// hashes) that check_match accepts, or -1.  rv: the version asked for, its name at rv_name, or null for an unversioned
// lookup.  newest: DL_LOOKUP_RETURN_NEWEST (dlsym): an unversioned lookup counts a definition at versym index 2 or
// above as a versioned candidate, where a relocation counts index 3 or above.  name is read only in [0, len).
ED_HD int64_t lookup_name(const Object &d, const uint8_t *da, const uint8_t *name, uint32_t len, uint32_t gnu,
                          uint32_t sysv, const Ver *rv, const uint8_t *rv_name, bool newest) {
  if (d.status != ST_OK || !d.nbucket || !d.nhash) return -1;
  const Tables t = tables(d);
  const uint8_t *syms = da + t.sym, *dstr = da + t.str;
  const Ver *dver = reinterpret_cast<const Ver *>(da + t.ver);
  const bool versym = d.flags & F_VERSYM;
  const uint32_t multi = newest ? 2 : 3;
  int64_t versioned = -1;
  uint32_t num_versions = 0;
  // check_match without the binding test (do_lookup_x applies that to what check_match returns)
  auto check = [&](uint64_t i) -> bool {
    const uint64_t s = i * SYM;
    const uint32_t info = syms[s + 4], shndx = (uint32_t)rd(syms, s + 6, 2), type = info & 0xf;
    if ((rd(syms, s + 8, 8) == 0 && shndx != SHN_ABS && type != STT_TLS) || shndx == SHN_UNDEF) return false;
    if (!((1u << type) & ALLOWED_STT)) return false;
    const uint64_t nm = rd(syms, s, 4);
    // .dynstr's copy ends in a NUL one past str_len: the definition's name must end right after len bytes
    if (nm >= d.str_len || len > d.str_len - nm || !same(dstr + nm, name, len) || dstr[nm + len]) return false;
    if (!versym) return true;
    const uint32_t vs = (uint32_t)rd(da + t.versym, 2 * i, 2), ndx = vs & 0x7fff;
    if (rv) {
      const Ver *dv = ndx < d.nver && (dver[ndx].flags & 1) ? dver + ndx : nullptr;
      const uint32_t dh = dv ? dv->hash : 0;
      const bool name_eq = dv && dv->name_len == rv->name_len && same(dstr + dv->name, rv_name, rv->name_len);
      return !((dh != rv->hash || !name_eq) && ((rv->flags & 2) || dh || (vs & 0x8000)));
    }
    if (ndx >= multi) {  // an unversioned lookup: a non-default version counts only as the object's single one
      if (!(vs & 0x8000) && num_versions++ == 0) versioned = (int64_t)i;
      return false;
    }
    return true;
  };
  int64_t hit = -1;
  if (d.flags & F_GNU) {
    const uint8_t *h = da + t.hash;
    const uint64_t word = rd(h, 16 + 8ull * ((gnu / 64) & (d.bloom_words - 1)), 8);
    if (!((word >> (gnu % 64)) & (word >> ((gnu >> d.bloom_shift) % 64)) & 1)) return -1;
    const uint8_t *bucket = h + 16 + 8ull * d.bloom_words, *chain = bucket + 4ull * d.nbucket;
    for (uint64_t i = rd(bucket, 4ull * (gnu % d.nbucket), 4); i && i < d.nhash; i++) {
      const uint32_t c = (uint32_t)rd(chain, 4 * (i - d.symoffset), 4);
      if (((c ^ gnu) >> 1) == 0 && check(i)) {
        hit = (int64_t)i;
        break;
      }
      if (c & 1) break;
    }
  } else {
    const uint8_t *h = da + t.hash, *bucket = h + 8, *chain = bucket + 4ull * d.nbucket;
    uint64_t steps = 0;
    for (uint64_t i = rd(bucket, 4ull * (sysv % d.nbucket), 4); i && i < d.nhash && steps < d.nhash;
         i = rd(chain, 4 * i, 4), steps++)
      if (check(i)) {
        hit = (int64_t)i;
        break;
      }
  }
  if (hit < 0 && num_versions == 1) hit = versioned;
  if (hit < 0) return -1;
  const uint32_t bind = syms[hit * SYM + 4] >> 4, vis = syms[hit * SYM + 5] & 3;
  if (!(bind == STB_GLOBAL || bind == STB_WEAK || bind == STB_GNU_UNIQUE)) return -1;
  if (vis == 1 || vis == 2) return -1;  // STV_INTERNAL, STV_HIDDEN
  return hit;
}

// lookup_name for the reference r of o (arena block oa), as a relocation looks it up.  rv: ref_version(o, oa, r).
ED_HD int64_t lookup(const Object &d, const uint8_t *da, const Object &o, const uint8_t *oa, const Ref &r, const Ver *rv) {
  const uint8_t *ostr = oa + tables(o).str;
  return lookup_name(d, da, ostr + r.name, r.name_len, r.gnu, r.sysv, rv, rv ? ostr + rv->name : nullptr, false);
}

// find: the first object of scope[scope_off ..+ scope_len) (lb2_sym_query) that defines the name pool[name_off ..+
// name_len) for dlsym; Found {obj, sym, st_info, st_other, versym} of it, obj NOT_FOUND when none does
constexpr uint32_t NOT_FOUND = 0xffffffffu;
struct Query {
  uint32_t scope_off, scope_len, name_off, name_len;
};
struct Found {
  uint32_t obj, sym;
  uint8_t info, other;
  uint16_t versym;
};
// Found of the symbol sym of d (arena block da)
ED_HD Found found_at(uint32_t id, const Object &d, const uint8_t *da, uint32_t sym) {
  const Tables t = tables(d);
  const uint8_t *e = da + t.sym + (uint64_t)sym * SYM;
  return Found{id, sym, e[4], e[5], d.flags & F_VERSYM ? (uint16_t)rd(da + t.versym, 2ull * sym, 2) : (uint16_t)0};
}

}  // namespace elfs
}  // namespace lb2
