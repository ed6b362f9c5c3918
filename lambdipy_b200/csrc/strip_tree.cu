// strip_tree.cu -- lb2_strip_tree: the directory walk that stands where the reference runs
// `find ... -name "*.so" | xargs strip` (lambdipy/project_build.py:260), the clean-up lines next to it, and the
// streaming engine that strips the selected files in place.
#include "lb2_host.cuh"

#include <atomic>
#include <cerrno>
#include <condition_variable>
#include <mutex>
#include <thread>

#include <dirent.h>
#include <fcntl.h>
#include <regex.h>
#include <spawn.h>
#include <sys/stat.h>
#include <sys/wait.h>

extern char **environ;

static bool ends_with(const char *s, const char *suf) {
  size_t a = strlen(s), b = strlen(suf);
  return a >= b && memcmp(s + a - b, suf, b) == 0;
}

struct TreeFile { std::string path; uint64_t size; dev_t dev; ino_t ino; uint32_t times; };

// The sibling lines of the reference's script (/root/reference/lambdipy/project_build.py:256-259), done on
// the same directory walk when asked for (LB2_TREE_CLEANUP):
//   rm -rf ROOT/*.egg-info ; rm -rf ROOT/*.dist-info                  top level, shell glob (no dot files)
//   find ROOT/ -name __pycache__ | xargs rm -rf                        any depth, any type
//   find ROOT/ -name tests | grep -v "PATTERN" | xargs rm -rf          PATTERN: a grep basic regex on the path
//                                                                      line find prints ("*" keeps only paths
//                                                                      containing a literal asterisk)
// They run before the strip line, so shared objects under a removed directory are never stripped.
struct Cleanup {
  bool on = false;
  regex_t keep;          // grep -v pattern for `tests`
  bool have_keep = false;
  uint32_t n_removed = 0;
  ~Cleanup() { if (have_keep) regfree(&keep); }
};

// The `tests` line on one entry named tests: `line` is the path find prints for it.  grep reads the printed list line
// by line, so a path holding a newline never matches as a whole and is left alone.
static bool tests_removed(const Cleanup &cl, const std::string &line) {
  return line.find('\n') == std::string::npos && !(cl.have_keep && regexec(&cl.keep, line.c_str(), 0, nullptr, 0) == 0);
}

static int compile_keep(Cleanup &cl, const char *keep_regex, std::string *err) {
  if (keep_regex && *keep_regex) {
    if (regcomp(&cl.keep, keep_regex, REG_NOSUB) != 0) { if (err) *err = std::string("bad keep-tests pattern: ") + keep_regex; return LB2_E_ARG; }
    cl.have_keep = true;
  }
  return LB2_OK;
}

static void rm_rf(const std::string &p) {
  struct stat sb;
  if (lstat(p.c_str(), &sb) != 0) return;
  if (S_ISDIR(sb.st_mode)) {
    if (DIR *d = opendir(p.c_str())) {
      while (dirent *e = readdir(d)) {
        if (!strcmp(e->d_name, ".") || !strcmp(e->d_name, "..")) continue;
        rm_rf(p + "/" + e->d_name);
      }
      closedir(d);
    }
    rmdir(p.c_str());
  } else {
    unlink(p.c_str());
  }
}

// `find ROOT/ -name "*SUFFIX"`: every directory entry whose basename matches, of any type; find does
// not descend into symlinked directories.  What `strip` then does with each path decides the rest:
//   regular file           -> stripped in place: GNU strip 2.42 writes the new contents back INTO THE
//                             EXISTING INODE (smart_rename copies), so mode, owner and every other hard
//                             link of the file are kept -- `libfoo.so.1` hard-linked to `libfoo.so` ends up
//                             stripped too although its name does not match
//   symlink to a file      -> the TARGET is rewritten, the link stays
//   directory / dangling   -> strip fails -> xargs exits 123 -> the reference's script aborts
// An inode reached through k matching paths (symlinks or hard links) is stripped k times by the
// reference; `times` keeps k.  Paths are kept as found: open() follows the links like strip does.
// `shown` is the path as find would print it (ROOT as given + "/" + relative part): what grep sees.
static void walk(const std::string &dir, const std::string &shown, bool top, const char *suffix, Cleanup *cl,
                 std::vector<TreeFile> &files, lb2_tree_stats *st) {
  DIR *d = opendir(dir.c_str());
  if (!d) return;
  std::vector<std::string> names;
  while (dirent *e = readdir(d))
    if (strcmp(e->d_name, ".") && strcmp(e->d_name, "..")) names.push_back(e->d_name);
  closedir(d);
  for (const std::string &name : names) {
    const std::string p = dir + "/" + name, line = shown + name;
    struct stat lsb, sb;
    if (lstat(p.c_str(), &lsb) != 0) continue;
    if (cl && cl->on) {
      bool remove = false;
      if (top && name[0] != '.' && (ends_with(name.c_str(), ".egg-info") || ends_with(name.c_str(), ".dist-info"))) remove = true;
      else if (name == "__pycache__") remove = true;
      else if (name == "tests" && tests_removed(*cl, line)) remove = true;
      if (remove) { rm_rf(p); cl->n_removed++; continue; }
    }
    if (suffix && ends_with(name.c_str(), suffix)) {
      st->n_selected++;
      if (stat(p.c_str(), &sb) != 0 || !S_ISREG(sb.st_mode)) {
        st->n_failed++;  // directory, dangling link, device ...: strip errors out
      } else {
        if (S_ISLNK(lsb.st_mode)) st->n_skipped++;  // the link itself is left alone
        files.push_back({p, (uint64_t)sb.st_size, sb.st_dev, sb.st_ino, 1});
      }
    }
    if (S_ISDIR(lsb.st_mode)) walk(p, line + "/", false, suffix, cl, files, st);
  }
}

// `find ROOT/ ...` over the directory `root`, after the clean-up lines when `cleanup` is set.  LB2_E_IO: root is not a
// directory; LB2_E_ARG: bad keep pattern.  `err` (may be null) receives the reason.
static int walk_root(const char *root, const char *suffix, bool cleanup, const char *keep_regex, std::string *err,
                     std::vector<TreeFile> &files, lb2_tree_stats *st) {
  struct stat rsb;
  if (stat(root, &rsb) != 0 || !S_ISDIR(rsb.st_mode)) { if (err) *err = std::string("not a directory: ") + root; return LB2_E_IO; }
  std::string r = root;
  while (r.size() > 1 && r.back() == '/') r.pop_back();
  Cleanup cl;
  if (cleanup) {
    cl.on = true;
    if (int rc = compile_keep(cl, keep_regex, err)) return rc;
  }
  walk(r, r + "/", true, suffix, &cl, files, st);
  st->n_removed = cl.n_removed;
  return LB2_OK;
}

static void dedupe(std::vector<TreeFile> &files) {
  std::sort(files.begin(), files.end(), [](const TreeFile &a, const TreeFile &b) {
    if (a.dev != b.dev) return a.dev < b.dev;
    if (a.ino != b.ino) return a.ino < b.ino;
    return a.path < b.path;
  });
  size_t w = 0;
  for (size_t i = 0; i < files.size(); i++) {
    if (w && files[w - 1].dev == files[i].dev && files[w - 1].ino == files[i].ino) files[w - 1].times++;
    else files[w++] = files[i];
  }
  files.resize(w);
  std::sort(files.begin(), files.end(), [](const TreeFile &a, const TreeFile &b) { return a.path < b.path; });
}

static int host_strip(const std::string &p) {
  const char *argv[] = {"strip", p.c_str(), nullptr};
  pid_t pid;
  if (posix_spawnp(&pid, "strip", nullptr, nullptr, const_cast<char *const *>(argv), environ) != 0) return 127;
  int status = 0;
  while (waitpid(pid, &status, 0) < 0 && errno == EINTR) {}
  return WIFEXITED(status) ? WEXITSTATUS(status) : 128;
}

template <class F> static void parallel_for(size_t n, int threads, F f) {
  std::atomic<size_t> next{0};
  std::vector<std::thread> pool;
  threads = (int)std::max<size_t>(1, std::min<size_t>((size_t)std::max(threads, 1), n));
  for (int t = 0; t < threads; t++)
    pool.emplace_back([&] { for (size_t i; (i = next.fetch_add(1)) < n;) f(i); });
  for (auto &th : pool) th.join();
}

// ---- the streaming engine behind lb2_strip_tree ---------------------------------------------------
// File bytes travel   page cache --pread--> pinned slot --DMA--> HBM input arena   and back
//                     HBM output arena --DMA--> pinned slot --pwrite--> the file's existing inode.
// Pinned memory is only a ring of small slots (two per I/O worker, LB2_TREE_SLOT_MB each), so a
// one-shot `lambdipy build` does not pay for pinning the tree twice and a 100 GB tree needs no more
// host memory than a small one.  The tree is cut into batches of whole files (<= LB2_TREE_BATCH_MB of
// arena span; a larger file is a batch of its own) that alternate between two HBM buffer sets: while
// batch b is downloaded and written, batch b+1 is read and uploaded -- the same worker pool serves both.
struct Seg { uint32_t file; uint64_t file_off, len, slot_off; };
struct Slice { bool upload; uint8_t *dev; uint64_t len; uint32_t seg0, seg1; };

static void make_slices(bool upload, uint8_t *dev_base, const std::vector<uint32_t> &ids, const uint64_t *offs, const uint64_t *sizes,
                        uint64_t slot_bytes, std::vector<Seg> &segs, std::vector<Slice> &out) {
  // ids[k] occupies [offs[k], offs[k] + sizes[k]) of the device arena, ascending and disjoint.  A slice is
  // one contiguous DMA range of at most slot_bytes; padding between neighbouring files rides along, a
  // larger hole (files that took another route) starts a new slice.
  const size_t m = ids.size();
  size_t k = 0;
  uint64_t c = 0;  // bytes of file k already covered by earlier slices
  while (k < m) {
    if (sizes[k] == 0) { k++; c = 0; continue; }
    const uint64_t a = offs[k] + c, end = a + slot_bytes;
    Slice sl{upload, dev_base + a, 0, (uint32_t)segs.size(), 0};
    uint64_t last = a;
    while (k < m) {
      if (sizes[k] == 0) { k++; c = 0; continue; }
      const uint64_t fs = offs[k] + c, fe = offs[k] + sizes[k];
      if (fs >= end || fs - last > 65536) break;
      const uint64_t take = std::min(fe, end) - fs;
      segs.push_back({ids[k], c, take, fs - a});
      last = fs + take;
      if (last == fe) { k++; c = 0; } else { c += take; break; }  // slot full inside a big file
    }
    sl.seg1 = (uint32_t)segs.size();
    sl.len = last - a;
    out.push_back(sl);
  }
}

struct TreeWorker { cudaStream_t stream = nullptr; cudaEvent_t ev[2] = {nullptr, nullptr}; uint32_t k = 0; };

struct TreeEngine {
  uint8_t *h_ring = nullptr;
  uint64_t slot_bytes = 0;
  int n_workers = 0;
  std::vector<TreeWorker> workers;
  uint8_t *d_in[2] = {nullptr, nullptr}, *d_out[2] = {nullptr, nullptr};
  uint64_t cap_in[2] = {0, 0}, cap_out[2] = {0, 0};
};

void tree_engine_free(TreeEngine *e) {
  if (!e) return;
  for (auto &w : e->workers) {
    if (w.stream) cudaStreamDestroy(w.stream);
    for (auto &ev : w.ev) if (ev) cudaEventDestroy(ev);
  }
  if (e->h_ring) cudaFreeHost(e->h_ring);
  for (int k = 0; k < 2; k++) { cudaFree(e->d_in[k]); cudaFree(e->d_out[k]); }
  delete e;
}

static int tree_engine_prepare(lb2_ctx *ctx, uint64_t expected_bytes) {
  if (ctx->tree) return LB2_OK;
  TreeEngine *e = new TreeEngine();
  e->slot_bytes = std::max<uint64_t>(1, env_u64("LB2_TREE_SLOT_MB", 4)) << 20;
  const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
  int want = (int)env_u64("LB2_IO_THREADS", std::max(4u, std::min(32u, hw / 2)));
  want = std::max(want, 1);
  if (expected_bytes) want = (int)std::max<uint64_t>(2, std::min<uint64_t>((uint64_t)want, expected_bytes / (2 * e->slot_bytes) + 1));
  e->n_workers = want;
  NumaPreferred near_gpu(ctx->numa_node);
  cudaError_t err = cudaHostAlloc(&e->h_ring, (uint64_t)want * 2 * e->slot_bytes, cudaHostAllocDefault);
  if (err != cudaSuccess) { ctx->err = std::string("cudaHostAlloc(tree ring): ") + cudaGetErrorString(err); delete e; return LB2_E_CUDA; }
  e->workers.resize(want);
  for (auto &w : e->workers) {
    if (cudaStreamCreateWithFlags(&w.stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&w.ev[0], cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&w.ev[1], cudaEventDisableTiming) != cudaSuccess) {
      ctx->err = "cuda stream/event creation failed"; tree_engine_free(e); return LB2_E_CUDA;
    }
  }
  ctx->tree = e;
  return LB2_OK;
}

static bool pread_all(int fd, uint8_t *dst, uint64_t n, uint64_t off) {
  uint64_t got = 0;
  while (got < n) {
    ssize_t r = pread(fd, dst + got, n - got, (off_t)(off + got));
    if (r <= 0) { if (r < 0 && errno == EINTR) continue; return false; }
    got += (uint64_t)r;
  }
  return true;
}
static bool pwrite_all(int fd, const uint8_t *src, uint64_t n, uint64_t off) {
  uint64_t put = 0;
  while (put < n) {
    ssize_t r = pwrite(fd, src + put, n - put, (off_t)(off + put));
    if (r <= 0) { if (r < 0 && errno == EINTR) continue; return false; }
    put += (uint64_t)r;
  }
  return true;
}

extern "C" {

int lb2_tree_prepare(lb2_ctx *ctx, uint64_t expected_tree_bytes) {
  if (!ctx) return LB2_E_ARG;
  CK(cudaSetDevice(ctx->device));
  int rc = tree_engine_prepare(ctx, expected_tree_bytes);
  if (rc) return rc;
  // the batch workspaces are first-use costs too
  rc = ws_reserve(ctx, ctx->ws, 256, 1 << 16);
  if (rc) return rc;
  return ws_reserve(ctx, ctx->ws2, 256, 1 << 16);
}

int lb2_tree_cleanup(const char *root, const char *keep_tests_regex, uint32_t *n_removed) {
  if (!root) return LB2_E_ARG;
  std::vector<TreeFile> files;
  lb2_tree_stats st;
  memset(&st, 0, sizeof st);
  int rc = walk_root(root, nullptr, true, keep_tests_regex, nullptr, files, &st);
  if (rc) return rc;
  if (n_removed) *n_removed = st.n_removed;
  return LB2_OK;
}

int lb2_cleanup_tests_removed(const char *keep_tests_regex, const char *const *lines, uint32_t n, uint8_t *removed) {
  if (n && (!lines || !removed)) return LB2_E_ARG;
  Cleanup cl;
  if (int rc = compile_keep(cl, keep_tests_regex, nullptr)) return rc;
  for (uint32_t i = 0; i < n; i++) {
    if (!lines[i]) return LB2_E_ARG;
    removed[i] = tests_removed(cl, lines[i]) ? 1 : 0;
  }
  return LB2_OK;
}

int lb2_strip_tree(lb2_ctx *ctx, const char *root, const char *suffix, uint32_t flags, lb2_tree_stats *st_out) {
  return lb2_strip_tree_ex(ctx, root, suffix, flags, nullptr, st_out);
}

int lb2_strip_tree_ex(lb2_ctx *ctx, const char *root, const char *suffix, uint32_t flags, const char *keep_tests_regex,
                      lb2_tree_stats *st_out) {
  if (!ctx || !root || !suffix) { if (ctx) ctx->err = "NULL argument"; return LB2_E_ARG; }
  CK(cudaSetDevice(ctx->device));
  lb2_tree_stats st;
  memset(&st, 0, sizeof st);
  double t0 = now_s();
  std::vector<TreeFile> files;
  int rc = walk_root(root, suffix, (flags & LB2_TREE_CLEANUP) != 0, keep_tests_regex, &ctx->err, files, &st);
  if (rc) return rc;
  dedupe(files);
  const uint32_t n = (uint32_t)files.size();
  uint64_t tree_bytes = 0;
  for (auto &f : files) tree_bytes += f.size;
  st.walk_read_s = now_s() - t0;
  if (!n) { if (st_out) *st_out = st; return LB2_OK; }
  rc = tree_engine_prepare(ctx, tree_bytes);
  if (rc) return rc;
  TreeEngine &E = *ctx->tree;
  const bool dry = (flags & LB2_TREE_DRY_RUN) != 0;

  // ---- batches of whole files
  const uint64_t batch_bytes = std::max<uint64_t>(1, env_u64("LB2_TREE_BATCH_MB", 1024)) << 20;
  struct Batch { uint32_t f0, f1; uint64_t span; };
  std::vector<Batch> batches;
  std::vector<uint64_t> off(n + 1), sizes(n), out_off(n + 1), out_sizes(n);  // offsets are relative to the batch's arena
  std::vector<int32_t> status(n, LB2_ST_MALFORMED);
  for (uint32_t f = 0; f < n;) {
    uint64_t pos = 0;
    uint32_t g = f;
    while (g < n && (g == f || pos + ((files[g].size + 255) & ~255ull) <= batch_bytes)) {
      off[g] = pos; sizes[g] = files[g].size; pos += (files[g].size + 255) & ~255ull; g++;
    }
    batches.push_back({f, g, pos});
    f = g;
  }

  // ---- worker pool: one task queue served by n_workers threads, each with two pinned slots + a stream
  std::vector<Seg> segs;
  std::vector<Slice> queue;
  std::atomic<size_t> q_next{0}, q_done{0};
  size_t q_end = 0;
  std::mutex mu;
  std::condition_variable cv_work, cv_done;
  bool quit = false;
  std::atomic<int> io_fail{0};
  std::atomic<uint64_t> ns_read{0}, ns_write{0}, ns_dma{0};  // summed over workers: where the I/O threads spend their time
  auto now_ns = [] { return (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  std::vector<std::atomic<int>> read_bad(n), write_bad(n);
  std::vector<std::atomic<uint32_t>> segs_left(n);
  for (uint32_t i = 0; i < n; i++) { read_bad[i] = 0; write_bad[i] = 0; segs_left[i] = 0; }
  std::atomic<uint32_t> n_gpu{0}, n_failed{0}, n_skipped{0};
  std::atomic<uint64_t> in_b{0}, out_b{0};
  std::vector<uint64_t> final_size(n, 0);

  auto finish_file = [&](uint32_t i) {
    // every piece of the new contents is in the inode: cut the old tail off
    bool ok = write_bad[i] == 0;
    if (ok && final_size[i] != files[i].size) ok = truncate(files[i].path.c_str(), (off_t)final_size[i]) == 0;
    if (ok) { n_gpu++; in_b += files[i].size; out_b += final_size[i]; }
    else n_failed++;
  };
  auto run_slice = [&](TreeWorker &w, int widx, const Slice &sl) {
    uint8_t *slot = E.h_ring + ((uint64_t)widx * 2 + (w.k & 1)) * E.slot_bytes;
    cudaEvent_t ev = w.ev[w.k & 1];
    w.k++;
    if (sl.upload) {
      uint64_t t0 = now_ns();
      cudaEventSynchronize(ev);  // the DMA that last read this slot has finished
      uint64_t t1 = now_ns();
      for (uint32_t q = sl.seg0; q < sl.seg1; q++) {
        const Seg &sg = segs[q];
        int fd = open(files[sg.file].path.c_str(), O_RDONLY | O_CLOEXEC);
        if (fd < 0 || !pread_all(fd, slot + sg.slot_off, sg.len, sg.file_off)) { read_bad[sg.file]++; io_fail++; }
        if (fd >= 0) close(fd);
      }
      uint64_t t2 = now_ns();
      cudaMemcpyAsync(sl.dev, slot, sl.len, cudaMemcpyHostToDevice, w.stream);
      cudaEventRecord(ev, w.stream);
      ns_dma += (t1 - t0) + (now_ns() - t2); ns_read += t2 - t1;
    } else {
      uint64_t t0 = now_ns();
      cudaMemcpyAsync(slot, sl.dev, sl.len, cudaMemcpyDeviceToHost, w.stream);
      cudaEventRecord(ev, w.stream);
      if (cudaEventSynchronize(ev) != cudaSuccess) io_fail++;
      uint64_t t1 = now_ns();
      ns_dma += t1 - t0;
      const uint64_t tw0 = t1;
      for (uint32_t q = sl.seg0; q < sl.seg1; q++) {
        const Seg &sg = segs[q];
        // no O_TRUNC, no temp file: the bytes go into the pages the file already has (see walk())
        int fd = open(files[sg.file].path.c_str(), O_WRONLY | O_CLOEXEC);
        if (fd < 0 || !pwrite_all(fd, slot + sg.slot_off, sg.len, sg.file_off)) write_bad[sg.file]++;
        if (fd >= 0) close(fd);
        if (--segs_left[sg.file] == 0) finish_file(sg.file);
      }
      ns_write += now_ns() - tw0;
    }
  };
  std::vector<std::thread> pool;
  for (int wi = 0; wi < E.n_workers; wi++)
    pool.emplace_back([&, wi] {
      cudaSetDevice(ctx->device);
      TreeWorker &w = E.workers[wi];
      for (;;) {
        size_t idx;
        {
          std::unique_lock<std::mutex> lk(mu);
          cv_work.wait(lk, [&] { return quit || q_next.load() < q_end; });
          if (q_next.load() >= q_end) { if (quit) return; continue; }
          idx = q_next.fetch_add(1);
        }
        run_slice(w, wi, queue[idx]);
        if (q_done.fetch_add(1) + 1 == q_end) { std::lock_guard<std::mutex> lk(mu); cv_done.notify_all(); }
      }
    });
  auto submit_and_wait = [&](std::vector<Slice> &a, std::vector<Slice> &b) {
    // interleave the two task lists so that downloads of batch b and uploads of batch b+1 overlap
    {
      std::lock_guard<std::mutex> lk(mu);
      size_t i = 0, j = 0;
      while (i < a.size() || j < b.size()) {
        if (i < a.size()) queue.push_back(a[i++]);
        if (j < b.size()) queue.push_back(b[j++]);
      }
      q_end = queue.size();
    }
    cv_work.notify_all();
    std::unique_lock<std::mutex> lk(mu);
    cv_done.wait(lk, [&] { return q_done.load() >= q_end; });
  };
  auto stop_pool = [&] {
    { std::lock_guard<std::mutex> lk(mu); quit = true; }
    cv_work.notify_all();
    for (auto &th : pool) th.join();
  };

  auto upload_slices = [&](size_t bi, std::vector<Slice> &out) -> int {
    const Batch &b = batches[bi];
    const int set = (int)(bi & 1);
    if (E.cap_in[set] < b.span + 256) CK(regrow(&E.d_in[set], E.cap_in[set], b.span + 256));
    std::vector<uint32_t> ids(b.f1 - b.f0);
    for (uint32_t i = b.f0; i < b.f1; i++) ids[i - b.f0] = i;
    make_slices(true, E.d_in[set], ids, off.data() + b.f0, sizes.data() + b.f0, E.slot_bytes, segs, out);
    return LB2_OK;
  };

  std::vector<void *> tmp_dev;  // outputs of the re-strip passes, freed at the end
  std::vector<Slice> up, down, none;
  double t_gpu = 0, t_io0 = now_s();
  // (a lambda so that every CUDA error path still reaches stop_pool() below)
  auto run_batches = [&]() -> int {
  int rc = upload_slices(0, up);
  if (rc == LB2_OK) submit_and_wait(up, none);
  for (size_t bi = 0; bi < batches.size() && rc == LB2_OK; bi++) {
    const Batch &b = batches[bi];
    const int set = (int)(bi & 1);
    const uint32_t m = b.f1 - b.f0;
    bool bad_read = false;
    for (uint32_t i = b.f0; i < b.f1; i++) bad_read |= read_bad[i] != 0;
    if (bad_read) { ctx->err = "could not read some selected files"; rc = LB2_E_IO; break; }
    // ---- kernels on the batch, inputs in HBM
    const double tg = now_s();
    for (auto &w : E.workers) { CK(cudaStreamWaitEvent(ctx->stream, w.ev[0], 0)); CK(cudaStreamWaitEvent(ctx->stream, w.ev[1], 0)); }
    const uint64_t want_out = b.span + (uint64_t)m * 4096 + (16u << 20);
    if (E.cap_out[set] < want_out) CK(regrow(&E.d_out[set], E.cap_out[set], want_out));
    Workspace &ws = set ? ctx->ws2 : ctx->ws;
    lb2_stats bst;
    rc = enqueue_batch(ctx, ws, E.d_in[set], off.data() + b.f0, sizes.data() + b.f0, m, E.d_out[set], E.cap_out[set], flags & 0xffu, ctx->stream, true);
    if (rc == LB2_OK) rc = collect_batch(ctx, ws, out_off.data() + b.f0, out_sizes.data() + b.f0, status.data() + b.f0, &bst);
    if (rc == LB2_E_CAPACITY)
      rc = redo_grown(ctx, ws, E.d_in[set], off.data() + b.f0, sizes.data() + b.f0, m, E.d_out[set], E.cap_out[set], flags & 0xffu,
                      ctx->stream, out_off.data() + b.f0, out_sizes.data() + b.f0, status.data() + b.f0, &bst);
    if (rc) break;
    st.batch.n_files += m;
    add_stats(st.batch, bst);
    // ---- inodes the reference strips more than once (several matching names): further passes run on
    //      the previous pass's output, still in HBM (strip is not idempotent on a few note layouts)
    std::vector<uint8_t *> src_base(m, E.d_out[set]);
    std::vector<uint64_t> src_off(out_off.begin() + b.f0, out_off.begin() + b.f1);
    for (uint32_t pass = 1; rc == LB2_OK; pass++) {
      std::vector<uint32_t> again;
      for (uint32_t i = b.f0; i < b.f1; i++) if (files[i].times > pass && status[i] == LB2_ST_OK) again.push_back(i);
      if (again.empty()) break;
      const uint32_t k2 = (uint32_t)again.size();
      std::vector<uint64_t> off2(k2 + 1), sz2(k2), ooff2(k2 + 1), osz2(k2);
      std::vector<int32_t> st2(k2);
      uint64_t p2 = 0;
      for (uint32_t k = 0; k < k2; k++) { off2[k] = p2; sz2[k] = out_sizes[again[k]]; p2 += (sz2[k] + 255) & ~255ull; }
      off2[k2] = p2;
      uint8_t *d_in2 = nullptr, *d_out2 = nullptr;
      const uint64_t cap2 = p2 + (uint64_t)k2 * 4096 + (64u << 20);
      CK(cudaMalloc(&d_in2, p2 + 256));
      tmp_dev.push_back(d_in2);
      CK(cudaMalloc(&d_out2, cap2));
      tmp_dev.push_back(d_out2);
      for (uint32_t k = 0; k < k2; k++) {
        const uint32_t i = again[k];
        CK(cudaMemcpyAsync(d_in2 + off2[k], src_base[i - b.f0] + src_off[i - b.f0], sz2[k], cudaMemcpyDeviceToDevice, ctx->stream));
      }
      lb2_stats b2;
      rc = enqueue_batch(ctx, ws, d_in2, off2.data(), sz2.data(), k2, d_out2, cap2, flags & 0xffu, ctx->stream, true);
      if (rc == LB2_OK) rc = collect_batch(ctx, ws, ooff2.data(), osz2.data(), st2.data(), &b2);
      if (rc == LB2_E_CAPACITY) { rc = LB2_OK; for (auto &x : st2) x = LB2_ST_UNSUPPORTED_LAYOUT; }  // hand them to the host strip
      if (rc) break;
      for (uint32_t k = 0; k < k2; k++) {
        const uint32_t i = again[k];
        status[i] = st2[k];
        if (st2[k] != LB2_ST_OK) continue;
        src_base[i - b.f0] = d_out2; src_off[i - b.f0] = ooff2[k]; out_sizes[i] = osz2[k];
      }
    }
    if (rc) break;
    t_gpu += now_s() - tg;
    // ---- download + write this batch, read + upload the next one
    down.clear(); up.clear();
    if (!dry) {
      // group by source buffer so that slices stay contiguous DMA ranges
      std::vector<uint8_t *> bases;
      for (uint32_t i = 0; i < m; i++) if (std::find(bases.begin(), bases.end(), src_base[i]) == bases.end()) bases.push_back(src_base[i]);
      for (uint8_t *base : bases) {
        std::vector<std::pair<uint64_t, uint32_t>> ord;
        for (uint32_t i = 0; i < m; i++)
          if (src_base[i] == base && status[b.f0 + i] == LB2_ST_OK) ord.push_back({src_off[i], b.f0 + i});
        std::sort(ord.begin(), ord.end());
        std::vector<uint32_t> ids;
        std::vector<uint64_t> o2, s2;
        for (auto &pr : ord) { ids.push_back(pr.second); o2.push_back(pr.first); s2.push_back(out_sizes[pr.second]); }
        const size_t seg_before = segs.size();
        make_slices(false, base, ids, o2.data(), s2.data(), E.slot_bytes, segs, down);
        for (size_t q = seg_before; q < segs.size(); q++) segs_left[segs[q].file]++;
        for (auto &pr : ord) {
          final_size[pr.second] = out_sizes[pr.second];
          if (out_sizes[pr.second] == 0) finish_file(pr.second);  // (cannot happen for a valid ELF; keeps the accounting total)
        }
      }
    } else {
      for (uint32_t i = b.f0; i < b.f1; i++) if (status[i] == LB2_ST_OK) { n_gpu++; in_b += files[i].size; out_b += out_sizes[i]; }
    }
    if (bi + 1 < batches.size()) rc = upload_slices(bi + 1, up);
    if (rc) break;
    submit_and_wait(down, up);
  }
  return rc;
  };
  rc = run_batches();
  stop_pool();
  cudaStreamSynchronize(ctx->stream);
  for (void *p : tmp_dev) cudaFree(p);
  st.gpu_s = t_gpu;
  st.read_cpu_s = ns_read.load() * 1e-9; st.write_cpu_s = ns_write.load() * 1e-9; st.dma_wait_s = ns_dma.load() * 1e-9;
  st.io_threads = (uint32_t)E.n_workers; st.n_batches = (uint32_t)batches.size();
  st.write_s = now_s() - t_io0 - t_gpu;  // read/upload and download/write overlap: I/O wall time next to the kernels
  if (rc) { if (st_out) *st_out = st; return rc; }

  t0 = now_s();
  std::vector<uint32_t> fallback;
  for (uint32_t i = 0; i < n; i++) if (status[i] != LB2_ST_OK) fallback.push_back(i);
  std::atomic<uint32_t> n_fb{0};
  parallel_for(fallback.size(), E.n_workers, [&](size_t k) {
    const uint32_t i = fallback[k];
    const bool non_elf = status[i] == LB2_ST_NOT_ELF;
    if (non_elf && (flags & LB2_TREE_TOLERATE_NON_ELF)) { n_skipped++; return; }
    if ((flags & LB2_TREE_FALLBACK_HOST_STRIP) && !dry) {
      // the reference's own tool decides (and fails the build exactly when the reference would)
      bool ok = true;
      for (uint32_t q = 0; q < files[i].times && ok; q++) ok = host_strip(files[i].path) == 0;
      if (ok) n_fb++; else n_failed++;
    } else {
      n_failed++;
    }
  });
  st.fallback_s = now_s() - t0;
  st.n_gpu = n_gpu; st.n_fallback = n_fb; st.n_failed += n_failed; st.n_skipped += n_skipped;
  st.in_bytes = in_b; st.out_bytes = out_b;
  if (st_out) *st_out = st;
  return LB2_OK;
}

}  // extern "C"
