// deps_emu.cpp -- TEST HARNESS: runs the PRODUCT's parse of dynamic sections (lambdipy_b200/csrc/elf_deps.cuh) on the
// CPU, one thread standing in for the warp of lb2_elf_deps_count_kernel / lb2_elf_deps_write_kernel: the same count
// pass, exclusive scan and write pass.  It is NOT a CPU fallback: it lives under tests/, is built only by the tests
// and is never loaded by lambdipy_b200/.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../lambdipy_b200/csrc/elf_deps.cuh"

using namespace lb2::elfd;

extern "C" {

// objects: n Object (lb2_elf_object); *records / *pool: the records and strings of all objects (free both with
// lb2emu_free); *n_records, *pool_bytes their sizes
int lb2emu_elf_deps(const uint8_t *const *ptrs, const uint64_t *sizes, uint32_t n, Object *objects, Record **records,
                    uint64_t *n_records, uint8_t **pool, uint64_t *pool_bytes) {
  SerialLanes lanes;
  uint64_t total_rec = 0, total_pool = 0;
  for (uint32_t i = 0; i < n; i++) {
    Count c;
    uint16_t machine, type;
    const int32_t st = parse(lanes, ptrs[i], sizes[i], c, machine, type);
    const bool ok = st == ST_OK;
    objects[i] = Object{st, machine, type, (uint32_t)total_rec, ok ? c.n : 0, total_pool, ok ? c.pool : 0};
    total_rec += objects[i].n_records;
    total_pool += objects[i].pool_len;
  }
  // exact sizes: the sanitizer build sees any write past them
  Record *rec = (Record *)malloc(sizeof(Record) * total_rec + 1);
  uint8_t *pl = (uint8_t *)malloc(total_pool + 1);
  for (uint32_t i = 0; i < n; i++) {
    if (objects[i].status != ST_OK || !objects[i].n_records) continue;
    Write w{rec + objects[i].first_record, pl, objects[i].pool_off, objects[i].n_records, objects[i].pool_len};
    uint16_t machine, type;
    parse(lanes, ptrs[i], sizes[i], w, machine, type);
    if (w.n != objects[i].n_records || w.used != objects[i].pool_len) {
      free(rec);
      free(pl);
      return -1;  // the two passes disagree
    }
  }
  *records = rec;
  *n_records = total_rec;
  *pool = pl;
  *pool_bytes = total_pool;
  return 0;
}

void lb2emu_free(void *p) { free(p); }
}

#ifdef LB2EMU_MAIN
// The sanitizer build (-fsanitize=address,undefined): every file named on the command line is read into a buffer of
// exactly its size and all of them are parsed in one batch; one line per file: status, records, pool bytes.
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
  std::vector<Object> obj(n + 1);
  Record *rec;
  uint8_t *pool;
  uint64_t nr, np;
  if (lb2emu_elf_deps(ptrs.data(), sizes.data(), n, obj.data(), &rec, &nr, &pool, &np)) return 4;
  for (uint32_t i = 0; i < n; i++) printf("%d %u %llu\n", obj[i].status, obj[i].n_records, (unsigned long long)obj[i].pool_len);
  for (uint32_t i = 0; i < n; i++) free((void *)ptrs[i]);
  free(rec);
  free(pool);
  return 0;
}
#endif
