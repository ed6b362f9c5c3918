// syms_emu.cpp -- TEST HARNESS: runs the PRODUCT's symbol index, reference list and lookup
// (lambdipy_b200/csrc/elf_syms.cuh) on the CPU, one thread standing in for each warp of elf_syms.cu, in the same order
// of passes as lb2_syms_index / lb2_syms_resolve / lb2_syms_names.  It is NOT a CPU fallback: it lives under tests/,
// is built only by the tests and is never loaded by lambdipy_b200/.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../lambdipy_b200/csrc/elf_syms.cuh"

using namespace lb2::elfs;

struct Emu {
  std::vector<uint8_t *> blocks;  // exact sizes: the sanitizer build sees any access past them
  std::vector<Object> objs;
};

extern "C" {

Emu *lb2emu_syms_create() { return new Emu; }

void lb2emu_syms_destroy(Emu *s) {
  for (uint8_t *b : s->blocks) free(b);
  delete s;
}

// lb2_syms_index's passes: count, place, write, mark, count references, place, write references
int lb2emu_syms_index(Emu *s, const uint8_t *const *ptrs, const uint64_t *sizes, uint32_t n, uint32_t *ids, Object *objects) {
  SerialLanes lanes;
  for (uint32_t i = 0; i < n; i++) {
    CountVer cv;
    Object o;
    const int32_t st = index(lanes, ptrs[i], sizes[i], o, cv);
    if (st != ST_OK) o = Object{};
    o.status = st;
    if (st == ST_OK) {
      uint8_t *a = (uint8_t *)calloc(tables(o).end, 1);
      s->blocks.push_back(a);
      o.arena = (uint64_t)a;
      const Tables t = tables(o);
      WriteVer wv{(Ver *)(a + t.ver), o.nver, true};
      Object again;
      index(lanes, ptrs[i], sizes[i], again, wv);
      memcpy(a + t.sym, ptrs[i] + o.sym_off, (uint64_t)o.nsyms * SYM);
      if (o.flags & F_VERSYM) memcpy(a + t.versym, ptrs[i] + o.versym_off, 2ull * o.nsyms);
      if (o.hash_len) memcpy(a + t.hash, ptrs[i] + o.hash_off, o.hash_len);
      if (o.str_len) memcpy(a + t.str, ptrs[i] + o.str_off, o.str_len);
      uint32_t *bits = (uint32_t *)(a + t.bits);
      for (uint64_t k = 0; k < o.rela_n + o.plt_n; k++) {
        const int64_t sy = mark(ptrs[i], o, a, k);
        if (sy >= 0) bits[sy / 32] |= 1u << (sy % 32);
        else if (sy == -2) o.flags |= F_BAD_REL;
      }
      uint32_t cnt = 0;
      bool bad = false;
      for (uint32_t sy = 0; sy < o.nsyms; sy++)
        if (bits[sy / 32] >> (sy % 32) & 1) {
          Ref r;
          bad |= !make_ref(o, a, sy, r);
          cnt++;
        }
      if (bad || (o.flags & F_BAD_REL)) {
        o.status = ST_MALFORMED;
        o.nrefs = 0;
      } else {
        o.nrefs = cnt;
      }
      if (o.nrefs) {
        Ref *refs = (Ref *)malloc(sizeof(Ref) * o.nrefs);
        s->blocks.push_back((uint8_t *)refs);
        o.refs = (uint64_t)refs;
        uint32_t k = 0;
        for (uint32_t sy = 0; sy < o.nsyms; sy++)
          if (bits[sy / 32] >> (sy % 32) & 1) make_ref(o, a, sy, refs[k++]);
      }
    }
    ids[i] = (uint32_t)s->objs.size();
    s->objs.push_back(o);
    objects[i] = o;
  }
  return 0;
}

// object id's references (nrefs of them)
const Ref *lb2emu_syms_refs(Emu *s, uint32_t id) { return (const Ref *)s->objs[id].refs; }

// lb2_syms_resolve: the warp's 32-entry ballot is the first defining entry in scope order
int lb2emu_syms_resolve(Emu *s, const Job *jobs, uint32_t n_jobs, const uint32_t *scope, const uint8_t *cls,
                        uint32_t *counts, Miss *miss, uint32_t max_miss, uint32_t *n_miss, uint64_t *lookups) {
  *n_miss = 0;
  *lookups = 0;
  for (uint32_t j = 0; j < n_jobs; j++) {
    counts[3 * j] = counts[3 * j + 1] = counts[3 * j + 2] = 0;
    const Object &o = s->objs[jobs[j].obj];
    const uint8_t *oa = (const uint8_t *)o.arena;
    for (uint32_t k = 0; k < o.nrefs; k++) {
      const Ref r = ((const Ref *)o.refs)[k];
      const Ver *rv = ref_version(o, oa, r);
      uint32_t found = jobs[j].scope_len;
      for (uint32_t e = 0; e < jobs[j].scope_len && found == jobs[j].scope_len; e++) {
        const Object &d = s->objs[scope[jobs[j].scope_off + e]];
        if (lookup(d, (const uint8_t *)d.arena, o, oa, r, rv) >= 0) found = e;
      }
      *lookups += found < jobs[j].scope_len ? found + 1 : jobs[j].scope_len;
      if (found < jobs[j].scope_len)
        counts[3 * j + cls[scope[jobs[j].scope_off + found]]]++;
      else if (!r.weak) {
        if (*n_miss < max_miss) miss[*n_miss] = Miss{j, k};
        ++*n_miss;
      }
    }
  }
  return *n_miss > max_miss ? -3 : 0;
}

// lb2_syms_names for one miss: name, version, file, each with its NUL, into out (cap bytes); the bytes needed
uint64_t lb2emu_syms_name(Emu *s, const Job *jobs, Miss m, char *out, uint64_t cap) {
  const Object &o = s->objs[jobs[m.job].obj];
  const uint8_t *a = (const uint8_t *)o.arena, *str = a + tables(o).str;
  const Ref r = ((const Ref *)o.refs)[m.ref];
  const Ver *v = ref_version(o, a, r);
  const uint8_t *p[3] = {str + r.name, v ? str + v->name : str, v && v->file != NO_STR ? str + v->file : str};
  const uint64_t l[3] = {r.name_len, v ? v->name_len : 0u, v && v->file != NO_STR ? v->file_len : 0u};
  const uint64_t need = l[0] + l[1] + l[2] + 3;
  if (need > cap) return need;
  for (int k = 0; k < 3; k++) {
    memcpy(out, p[k], l[k]);
    out[l[k]] = 0;
    out += l[k] + 1;
  }
  return need;
}
}

#ifdef LB2EMU_MAIN
// The sanitizer build (-fsanitize=address,undefined): every file named on the command line is read into a buffer of
// exactly its size and indexed in one batch; then each object's references are resolved in the scope of all of them.
// One line per file: status, symbols, references, misses.
int main(int argc, char **argv) {
  const uint32_t n = argc - 1;
  std::vector<const uint8_t *> ptrs(n + 1);
  std::vector<uint64_t> sizes(n + 1);
  for (uint32_t i = 0; i < n; i++) {
    FILE *f = fopen(argv[i + 1], "rb");
    if (!f) return 3;
    fseek(f, 0, SEEK_END);
    sizes[i] = ftell(f);
    fseek(f, 0, SEEK_SET);
    uint8_t *b = (uint8_t *)malloc(sizes[i] ? sizes[i] : 1);
    if (fread(b, 1, sizes[i], f) != sizes[i]) return 3;
    fclose(f);
    ptrs[i] = b;
  }
  Emu *s = lb2emu_syms_create();
  std::vector<uint32_t> ids(n + 1);
  std::vector<Object> obj(n + 1);
  lb2emu_syms_index(s, ptrs.data(), sizes.data(), n, ids.data(), obj.data());
  for (uint32_t i = 0; i < n; i++) free((void *)ptrs[i]);  // the arena must not need them
  std::vector<Job> jobs(n + 1);
  std::vector<uint32_t> scope(n + 1);
  std::vector<uint8_t> cls(n + 1, 0);
  for (uint32_t i = 0; i < n; i++) {
    jobs[i] = Job{ids[i], 0, n, 0};
    scope[i] = ids[i];
  }
  std::vector<uint32_t> counts(3 * n + 3);
  uint32_t cap = 1 << 20, n_miss;
  uint64_t lookups;
  std::vector<Miss> miss(cap);
  lb2emu_syms_resolve(s, jobs.data(), n, scope.data(), cls.data(), counts.data(), miss.data(), cap, &n_miss, &lookups);
  std::vector<uint32_t> per(n + 1, 0);
  char buf[1 << 16];
  for (uint32_t k = 0; k < n_miss && k < cap; k++) {
    per[miss[k].job]++;
    lb2emu_syms_name(s, jobs.data(), miss[k], buf, sizeof buf);
  }
  for (uint32_t i = 0; i < n; i++) printf("%d %u %u %u\n", obj[i].status, obj[i].nsyms, obj[i].nrefs, per[i]);
  lb2emu_syms_destroy(s);
  return 0;
}
#endif
