"""Will the shared objects of a Lambda zip load there?  `check_zip(zip_path)` reads the dynamic sections of every
shared object the zip's `import`s would load, on the GPU where the zip reader leaves the decoded bytes
(lb2_elf_deps), and restates the dynamic loader's search for each one.

    python -m lambdipy_b200.deps ZIP [--mount DIR] [--arch x86_64|arm64] [--provided NAME]...
                                     [--max-version GLIBC_2.26]... [--ld-library-path P] [--json]
                                     [--symbols [--interpreter FILE]... [--runtime-lib DIR]...] [--python 3.N]

A layer fails at the first `import` when a shared object cannot load: a DT_NEEDED library that neither the zip nor
the runtime has, a symbol version newer than the runtime's, an object for the other architecture.  The check finds
these before the upload instead of in a traceback afterwards.

Roots are the members the strip line selects (a regular file whose basename ends in ".so"); member `a/b.so` lies at
`mount/a/b.so` (/var/task for a function bundle, /opt for a layer written with prefix="python/").  For each root the
closure is what `dlopen` of that root would load, restated from glibc's _dl_map_object: breadth first over DT_NEEDED
in dynamic-array order; a name already matching an object of that closure (the name it was loaded by, or its
DT_SONAME) is that object; a name with a '/' is a path; otherwise the directories of DT_RPATH of the object and of its
loader chain (not when the object has DT_RUNPATH, and an object's DT_RPATH counts for nothing when it has DT_RUNPATH),
then `ld_library_path`, then the object's DT_RUNPATH, then the runtime's own libraries.  $ORIGIN, $LIB and $PLATFORM
are expanded against the path the object was found at.  Symlink members are followed inside the zip, up to 40 hops.

Members are decoded and parsed in rounds: the roots first, then whatever they reach inside the zip that has not been
parsed yet, and so on.  The GPU reader decodes each round (halving on a device too small); a member it does not take
is read by the stdlib and uploaded.

`provided` is the set of sonames the runtime image supplies from its own directories (/lib64, /usr/lib64, and the
loader's defaults).  The default -- glibc's libraries plus libgcc_s.so.1, libstdc++.so.6 and libz.so.1 -- is a guess
that nobody has checked against a Lambda image here; the report names every need that the list satisfied
(`provided_used`), so nothing is hidden behind it.

Deviations from the loader, each documented in DESIGN.md section 9.8: a candidate file is taken when it exists (glibc
also skips a candidate of the wrong ELF class or machine and searches on; here that is an `arch` problem); the
executable's own DT_RPATH, ld.so.cache entries beyond `provided`, libraries opened by `dlopen` at run time and the
effects of import order between roots are not modelled.

With symbols=True (--symbols) the check also looks up, on the GPU, every symbol that an object's relocations bind when
`dlopen` loads it with RTLD_NOW, as glibc's do_lookup_x and check_match do, in the scope of the interpreter's global
objects followed by the root's closure (lb2_syms_*; DESIGN.md section 9.9).  This finds the `undefined symbol` of an
extension module built against another version of a library the zip carries.  Only counts and the failed lookups come
back from the device.

With python="3.N" (--python) the check also restates CPython's import finder (importlib's PathFinder and FileFinder)
over the zip's tree on Lambda's sys.path and classes every `*.so` under it: an extension module the finder loads, a
file it shadows, a build for another Python (a `cpython-3M` / `pypy` tag the target does not load) or a library.
Each module's `PyInit_<name>` is looked up on the GPU as dlsym looks it up in the module's own load scope
(lb2_syms_find; DESIGN.md section 9.11).  This finds `No module named ...` of a wheel built for another Python and
`dynamic module does not define module export function` of a renamed extension before the upload.

The check runs over entries (check_entries): check_with builds them from a zip's central directory, and the layer
writers (layer.zip_build / zip_tarballs with check=...) from the entries of the zip they are about to write, with the
bytes they already hold on the device (DESIGN.md section 9.10)."""
import json
import os
import posixpath
import re
import stat
import sys
import zipfile

import ctypes as C

from . import _native as N
from . import zipfile_gpu as Z

LAMBDA_LD_LIBRARY_PATH = "/var/lang/lib:/lib64:/usr/lib64:/var/runtime:/var/runtime/lib:/var/task:/var/task/lib:/opt/lib"
LAMBDA_TASK_ROOT = "/var/task"      # the working directory of a Lambda function: relative names resolve there
RUNTIME_DIRS = ("/lib64", "/usr/lib64")  # where the runtime image keeps the `provided` libraries
DEFAULT_PROVIDED = frozenset([
    "ld-linux-x86-64.so.2", "libc.so.6", "libm.so.6", "libpthread.so.0", "libdl.so.2", "librt.so.1", "libutil.so.1",
    "libresolv.so.2", "libnsl.so.1", "libanl.so.1", "libmvec.so.1", "libgcc_s.so.1", "libstdc++.so.6", "libz.so.1"])
MACHINES = {"x86_64": 62, "arm64": 183}
PLATFORMS = {"x86_64": "x86_64", "arm64": "aarch64"}
STATUS_NAMES = {N.ELF_OK: "ok", N.ELF_NOT_ELF: "not ELF", N.ELF_UNSUPPORTED: "unsupported", N.ELF_STATIC: "static",
                N.ELF_MALFORMED: "malformed"}
SYMLINK_HOPS = 40
BATCH_BYTES = Z.BATCH_BYTES
_VERSION = re.compile(r"^([A-Za-z][A-Za-z0-9]*)_(\d+(?:\.\d+)*)$")
VER_FLG_WEAK = 2
CLASS_IN_ZIP, CLASS_RUNTIME, CLASS_INTERPRETER = 0, 1, 2  # where a reference's definition was found
PYTHON_VERSIONS = tuple("3.%d" % m for m in range(8, 15))
# Lambda's sys.path entries a zip can fill, in order, from AWS's runtime documentation (/var/task, then a layer's
# python/lib/python3.N/site-packages and python/); nobody has checked it against a runtime image here, so the report
# echoes it.  The runtime's own entries come after these and are not modelled.
LAMBDA_PYTHON_PATH = ("/var/task", "/opt/python/lib/python{version}/site-packages", "/opt/python")
TRIPLETS = {"x86_64": "x86_64-linux-gnu", "arm64": "aarch64-linux-gnu"}
_PY_TAG = re.compile(r"^([^.]+)\.((?:cpython-|pypy)[^.]*)\.so$")  # stem.TAG.so: an extension built for some Python


class GpuElfParser:
    """lb2_elf_deps over objects in device memory.  parse(refs): refs are (device address, size) pairs; returns
    [(status, machine, [(kind, flags, ref, name)])].  upload(data) puts a member the GPU reader did not take on the
    device until the next parse(); uploaded / downloaded count the bytes that crossed the bus."""

    def __init__(self, ctx):
        self._ctx, self._extra = ctx, []
        self.uploaded = self.downloaded = 0
        self._rec_cap, self._pool_cap = 1 << 12, 1 << 18
        self._stats = {"kernel_ms": 0.0, "objects": 0, "calls": 0}

    def _release(self):
        for p in self._extra:
            self._ctx.dev_free(p)
        self._extra = []

    def parse(self, refs):
        n = len(refs)
        if not n:
            self._release()
            return []
        ptrs = (C.c_uint64 * n)(*[a for a, _ in refs])
        sizes = (C.c_uint64 * n)(*[k for _, k in refs])
        objs, nr, npool, st = (N.ElfObject * n)(), C.c_uint32(), C.c_uint64(), N.ElfDepsStats()
        lib, ctx = self._ctx.lib, self._ctx
        while True:
            recs = (N.ElfRecord * self._rec_cap)()
            pool = C.create_string_buffer(self._pool_cap)
            rc = lib.lb2_elf_deps(ctx.h, ptrs, sizes, n, objs, recs, self._rec_cap, C.byref(nr), pool, self._pool_cap,
                                  C.byref(npool), C.byref(st))
            self._stats["kernel_ms"] += st.kernel_ms
            self.downloaded += st.bytes_down
            if rc == N.LB2_E_CAPACITY:
                self._rec_cap = max(self._rec_cap, nr.value)
                self._pool_cap = max(self._pool_cap, npool.value)
                continue
            ctx.check(rc)
            break
        self._release()
        self._stats["objects"] += n
        self._stats["calls"] += 1
        return decode(objs, recs, pool.raw[:npool.value])

    def upload(self, data):
        p = self._ctx.dev_alloc(max(len(data), 1))
        self._extra.append(p)
        if data:
            self._ctx.h2d(p, data, len(data))
        self.uploaded += len(data)
        return p, len(data)

    def stats(self):
        return dict(self._stats)

    def close(self):
        self._release()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class GpuSymbolResolver:
    """lb2_syms_* over objects in device memory, for a whole check: index(refs) copies each object's symbol tables
    into the resolver's device arena while the object is still there and returns [(id, status, references)];
    resolve(jobs, scope, classes) looks every reference of jobs' objects up in their scopes and returns ([(in_zip,
    runtime, interpreter) per job], [(job, reference) found nowhere, sorted]); names(jobs, misses) gives [(name, version,
    version file)] of misses; find(queries, scope) looks names up as dlsym does.  uploaded / downloaded count the
    bytes that crossed the bus."""

    def __init__(self, ctx):
        self._ctx, h = ctx, C.c_void_p()
        ctx.check(ctx.lib.lb2_syms_create(ctx.h, C.byref(h)))
        self._h = h
        self.uploaded = self.downloaded = 0
        self._miss_cap = 1 << 12
        self._stats = {"index_ms": 0.0, "refs_ms": 0.0, "resolve_ms": 0.0, "references": 0, "lookups": 0,
                       "find_ms": 0.0, "find_queries": 0}

    def _account(self, st):
        self.uploaded += st.bytes_up
        self.downloaded += st.bytes_down
        for k in ("index_ms", "refs_ms", "resolve_ms"):
            self._stats[k] += getattr(st, k)

    def index(self, refs):
        n = len(refs)
        if not n:
            return []
        ptrs = (C.c_uint64 * n)(*[a for a, _ in refs])
        sizes = (C.c_uint64 * n)(*[k for _, k in refs])
        ids, objs, st = (C.c_uint32 * n)(), (N.SymObject * n)(), N.SymsStats()
        rc = self._ctx.lib.lb2_syms_index(self._h, ptrs, sizes, n, ids, objs, C.byref(st))
        self._account(st)
        if rc == N.LB2_E_CAPACITY:  # the arena cannot grow by this batch: index it in halves
            if n == 1:
                raise Z.DeviceTooSmall("lb2_syms_index: no device memory for the symbol arena")
            return self.index(refs[:n // 2]) + self.index(refs[n // 2:])
        self._ctx.check(rc)
        self._stats["references"] += st.references
        return [(ids[i], objs[i].status, objs[i].nrefs) for i in range(n)]

    def resolve(self, jobs, scope, classes):
        nj, ns = len(jobs), len(scope)
        cj = (N.SymJob * max(nj, 1))(*[N.SymJob(o, off, ln, 0) for o, off, ln in jobs])
        cs = (C.c_uint32 * max(ns, 1))(*scope)
        cc = (C.c_uint8 * max(len(classes), 1))(*classes)
        counts, nm, st = (C.c_uint32 * max(3 * nj, 1))(), C.c_uint32(), N.SymsStats()
        while True:
            miss = (N.SymMiss * self._miss_cap)()
            rc = self._ctx.lib.lb2_syms_resolve(self._h, cj, nj, cs, ns, cc, counts, miss, self._miss_cap, C.byref(nm),
                                                C.byref(st))
            self._account(st)
            if rc == N.LB2_E_CAPACITY:
                self._miss_cap = max(2 * self._miss_cap, nm.value)
                continue
            self._ctx.check(rc)
            break
        self._stats["lookups"] += st.lookups
        return ([tuple(counts[3 * j:3 * j + 3]) for j in range(nj)],
                sorted((miss[i].job, miss[i].ref) for i in range(nm.value)))  # the kernel appends them in any order

    def names(self, jobs, misses):
        n = len(misses)
        if not n:
            return []
        cj = (N.SymJob * max(len(jobs), 1))(*[N.SymJob(o, off, ln, 0) for o, off, ln in jobs])
        cm = (N.SymMiss * n)(*[N.SymMiss(j, r) for j, r in misses])
        offs, need, st, cap = (C.c_uint64 * n)(), C.c_uint64(), N.SymsStats(), 64 * n
        while True:
            pool = C.create_string_buffer(cap)
            rc = self._ctx.lib.lb2_syms_names(self._h, cj, len(jobs), cm, n, offs, pool, cap, C.byref(need), C.byref(st))
            self._account(st)
            if rc == N.LB2_E_CAPACITY:
                cap = need.value
                continue
            self._ctx.check(rc)
            break
        raw = pool.raw
        return [tuple(x.decode("utf-8", "surrogateescape") for x in raw[offs[i]:].split(b"\0", 3)[:3]) for i in range(n)]

    def find(self, queries, scope):
        """dlsym of names in scopes: queries [(scope_off, scope_len, name bytes)] over scope (resolver ids) ->
        [(id of the first object defining it or None, symbol index, st_info, st_other, versym)]"""
        n = len(queries)
        if not n:
            return []
        cq, pool, found = find_arrays(queries)
        cs, st = (C.c_uint32 * max(len(scope), 1))(*scope), N.SymsStats()
        rc = self._ctx.lib.lb2_syms_find(self._h, cq, n, cs, len(scope), pool, len(pool), found, C.byref(st))
        self._ctx.check(rc)
        self.uploaded += st.bytes_up
        self.downloaded += st.bytes_down
        self._stats["find_ms"] += st.resolve_ms
        self._stats["find_queries"] += n
        return found_records(found, n)

    def stats(self):
        return dict(self._stats)

    def close(self):
        if self._h:
            self._ctx.lib.lb2_syms_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def find_arrays(queries):
    """(lb2_sym_query array, name pool bytes, lb2_sym_found array) of find's queries [(scope_off, scope_len, name)]"""
    cq, at = (N.SymQuery * max(len(queries), 1))(), 0
    for i, (off, ln, name) in enumerate(queries):
        cq[i] = N.SymQuery(off, ln, at, len(name))
        at += len(name)
    return cq, b"".join(name for _, _, name in queries), (N.SymFound * max(len(queries), 1))()


def found_records(found, n):
    """find's result of an lb2_sym_found array"""
    return [(None if f.obj == N.SYM_NOT_FOUND else f.obj, f.sym, f.info, f.other, f.versym) for f in found[:n]]


def decode(objs, recs, pool):
    """lb2_elf_object / lb2_elf_record arrays and the pool -> [(status, machine, [(kind, flags, ref, name)])]"""
    out = []
    for o in objs:
        rs = []
        for r in recs[o.first_record:o.first_record + o.n_records]:
            rs.append((r.kind, r.flags, r.ref, pool[r.off:r.off + r.len].decode("utf-8", "surrogateescape")))
        out.append((o.status, o.machine, rs))
    return out


class _Obj:
    """what the loader model needs of one parsed member (member: its entry's name)"""

    def __init__(self, member, status, machine, records):
        self.member, self.status, self.machine = member, status, machine
        self.soname = None
        self.needed, self.rpath, self.runpath, self.verdef, self.verneed = [], None, None, set(), []
        files = {}
        for i, (kind, flags, ref, name) in enumerate(records):
            if kind == N.ELF_REC_NEEDED:
                self.needed.append(name)
            elif kind == N.ELF_REC_SONAME:
                self.soname = name
            elif kind == N.ELF_REC_RPATH:
                self.rpath = name if self.rpath is None else self.rpath + ":" + name
            elif kind == N.ELF_REC_RUNPATH:
                self.runpath = name if self.runpath is None else self.runpath + ":" + name
            elif kind == N.ELF_REC_VERNEED_FILE:
                files[i] = name
            elif kind == N.ELF_REC_VERNEED_VERSION:
                self.verneed.append((files.get(ref, ""), name, bool(flags & VER_FLG_WEAK)))
            elif kind == N.ELF_REC_VERDEF:
                self.verdef.add(name)
        if self.runpath is not None:
            self.rpath = None  # glibc: DT_RPATH is ignored when DT_RUNPATH is present


class _Tree:
    """The zip as the file system under `mount`: {absolute path: key of a regular file | link target}, and the
    directories its paths imply.  entries [(key, name, link)]: an opaque key, the entry's name (a directory's ends in
    "/") and a symlink's target (None for a regular file or a directory)."""

    def __init__(self, entries, mount):
        self.mount = posixpath.normpath("/" + mount.strip("/")) if mount.strip("/") else "/"
        self.files, self.links, self.dirs, self.names = {}, {}, {self.mount}, {}
        self._children = None
        d = self.mount
        while d != "/":
            d = posixpath.dirname(d)
            self.dirs.add(d)
        for key, entry_name, link in entries:  # a repeated name: the last entry, as getinfo and extractall leave it
            self.names[key] = entry_name
            name = entry_name.rstrip("/")
            if not name:
                continue
            path = posixpath.normpath(posixpath.join(self.mount, name))
            d = posixpath.dirname(path)
            while d not in self.dirs:
                self.dirs.add(d)
                d = posixpath.dirname(d)
            self.files.pop(path, None)
            self.links.pop(path, None)
            if entry_name.endswith("/"):
                self.dirs.add(path)
            elif link is not None:
                self.links[path] = link
            else:
                self.files[path] = key

    def lookup(self, path):
        """the key of the regular file `path` ends at, symlinks followed, or None"""
        got = self._walk(path)
        return got[1] if got and got[0] == "file" else None

    def directory(self, path):
        """the directory `path` ends at, symlinks followed, or None"""
        got = self._walk(path)
        return got[1] if got and got[0] == "dir" else None

    def children(self, d):
        """the names in the directory d (a path directory() returned): files, links and directories"""
        if self._children is None:
            self._children = {}
            for p in list(self.files) + list(self.links) + list(self.dirs):
                if p != "/":
                    self._children.setdefault(posixpath.dirname(p), set()).add(posixpath.basename(p))
        return self._children.get(d, set())

    def _walk(self, path):
        """("file", key) or ("dir", its path) where `path` ends, symlinks followed, or None"""
        parts, i, cur, hops = [x for x in path.split("/") if x], 0, [], SYMLINK_HOPS
        while i < len(parts):
            comp = parts[i]
            if comp == ".":
                i += 1
                continue
            if comp == "..":
                cur = cur[:-1]
                i += 1
                continue
            p = "/" + "/".join(cur + [comp])
            if p in self.links:
                hops -= 1
                if hops < 0:
                    return None
                t = self.links[p]
                base = [] if t.startswith("/") else cur
                parts, i, cur = base + [x for x in t.split("/") if x] + parts[i + 1:], 0, []
                continue
            last = i + 1 == len(parts) or all(x in ("", ".") for x in parts[i + 1:])
            if p in self.files:
                return ("file", self.files[p]) if last else None
            if p not in self.dirs:
                return None
            cur.append(comp)
            i += 1
        return "dir", "/" + "/".join(cur)


def _version_key(v):
    return tuple(int(x) for x in v.split("."))


def _expand(dirs, origin, arch):
    out = []
    for d in dirs.split(":"):
        if d == "":
            d = LAMBDA_TASK_ROOT  # an empty entry is the working directory
        for token, value in (("ORIGIN", origin), ("LIB", "lib64"), ("PLATFORM", PLATFORMS[arch])):
            d = d.replace("${%s}" % token, value).replace("$" + token, value)
        out.append(d)
    return out


class _Model:
    """the loader's search for each root's closure over the objects parsed so far"""

    def __init__(self, tree, objs, arch, provided, ld_library_path):
        self.tree, self.objs, self.arch = tree, objs, arch
        self.provided = frozenset(provided)
        self.env = _expand(ld_library_path or "", LAMBDA_TASK_ROOT, arch) if ld_library_path else []

    def _find(self, name, obj_path, chain):
        """(how, path or None, key or None) for NEEDED `name` of the object at obj_path loaded through `chain`"""
        if "/" in name:
            path = posixpath.join(LAMBDA_TASK_ROOT, name)
            key = self.tree.lookup(path)
            return ("path", path, key) if key is not None else ("missing", None, None)
        obj = self.objs[chain[-1][1]]
        searches = []
        if obj.runpath is None:
            for p, key in reversed(chain):
                o = self.objs[key]
                if o.rpath is not None:
                    searches.append(("rpath", _expand(o.rpath, posixpath.dirname(p), self.arch)))
        searches.append(("ld_library_path", self.env))
        if obj.runpath is not None:
            searches.append(("runpath", _expand(obj.runpath, posixpath.dirname(obj_path), self.arch)))
        for how, dirs in searches:
            for d in dirs:
                if name in self.provided and posixpath.normpath(d) in RUNTIME_DIRS:
                    return "provided", None, None
                path = posixpath.join(d, name)
                key = self.tree.lookup(path)
                if key is not None:
                    return how, path, key
        return ("provided", None, None) if name in self.provided else ("missing", None, None)

    def closure(self, root_path, root_key):
        """(loaded [(path, key)] in load order, [(loader path, its key, name, how, path)], unparsed keys reached)"""
        loaded = [(root_path, root_key)]
        names = {root_key: {root_path}}
        loader = {root_key: None}
        provided_loaded = set()
        resolutions, pending = [], []
        q = 0
        while q < len(loaded):
            path, key = loaded[q]
            q += 1
            obj = self.objs.get(key)
            if obj is None:
                pending.append(key)
                continue
            if obj.status != N.ELF_OK:
                continue
            chain, z = [], key  # this object, its loader, and on up to the root
            while z is not None:
                chain.insert(0, (next(p for p, y in loaded if y == z), z))
                z = loader[z]
            for name in obj.needed:
                hit = next((y for p, y in loaded if name in names[y] or
                            (y in self.objs and self.objs[y].soname == name)), None)
                if hit is not None:
                    resolutions.append((path, key, name, "loaded", next(p for p, y in loaded if y == hit)))
                    names[hit].add(name)
                    continue
                if name in provided_loaded:
                    resolutions.append((path, key, name, "provided", None))
                    continue
                how, found, fkey = self._find(name, path, chain)
                if fkey is not None and fkey in names:  # the same file by another name: one object
                    names[fkey].add(name)
                    resolutions.append((path, key, name, how, next(p for p, y in loaded if y == fkey)))
                    continue
                resolutions.append((path, key, name, how, found))
                if how == "provided":
                    provided_loaded.add(name)
                elif fkey is not None:
                    loaded.append((found, fkey))
                    names[fkey] = {name, found}
                    loader[fkey] = key
        return loaded, resolutions, pending


CHECK_KEYS = ("mount", "arch", "provided", "max_versions", "ld_library_path", "symbols", "interpreter", "runtime_libs",
              "python")


class CheckFailed(Exception):
    """A layer writer's check found problems: report is what check_zip would return for the zip it did not write."""

    def __init__(self, report):
        first = report["problems"][0]
        super().__init__("%d problem(s), the first: %s: %s: %s" % (len(report["problems"]), first["object"],
                                                                   first["kind"], first["detail"]))
        self.report = report


def _ceilings(arch, max_versions):
    """{prefix: version key} of max_versions; ValueError for an unknown arch or a version that is not dotted"""
    if arch not in MACHINES:
        raise ValueError("arch=%r: expected one of %s" % (arch, ", ".join(MACHINES)))
    ceilings = {}
    for prefix, v in (max_versions or {}).items():
        if not re.fullmatch(r"\d+(?:\.\d+)*", str(v)):
            raise ValueError("max_versions[%r]=%r: expected a dotted version such as 2.26" % (prefix, v))
        ceilings[prefix] = _version_key(str(v))
    return ceilings


def check_options(check):
    """check_zip's keyword arguments in the dict `check`, refused as check_with refuses them: ValueError for a key that
    is not one of CHECK_KEYS, an unknown arch, a max_versions value that is not a dotted version or a python version
    that is not one of PYTHON_VERSIONS"""
    if not isinstance(check, dict):
        raise ValueError("check=%r: expected a dict of check_zip's keyword arguments" % (check,))
    unknown = sorted(set(check) - set(CHECK_KEYS))
    if unknown:
        raise ValueError("check: unknown key(s) %s; expected some of %s" % (", ".join(map(repr, unknown)),
                                                                         ", ".join(CHECK_KEYS)))
    _ceilings(check.get("arch", "x86_64"), check.get("max_versions"))
    python_version(check.get("python"))
    return dict(check)


def member_decoder(decoder, parser, members, batch_bytes=BATCH_BYTES):
    """The decode step of check_entries over zip members, members {key: (ZipInfo, (ZipFile, its open file, its size))}:
    a round's members go to the GPU reader in batches of about batch_bytes (Z.decode_members, halved on a device too
    small); a member the reader does not take is read by the stdlib and uploaded through the parser."""
    def decode(keys, consume):
        def part_done(part, decoded, whole):
            refs = []
            for key, zi, (zf, _, _) in part:
                status, ref = decoded.get(key, (Z.UNZIP_OK, None))
                if status != Z.UNZIP_OK:
                    raise Z.BadZipMember(zi.filename, {Z.UNZIP_BAD_DATA: "Invalid DEFLATE data", Z.UNZIP_BAD_CRC: "Bad CRC-32",
                                                       Z.UNZIP_WRONG_SIZE: "Wrong uncompressed size"}[status])
                refs.append(ref if ref is not None else parser.upload(zf.read(zi)))
            consume([key for key, _, _ in part], refs)

        uploaded, batch, cost = 0, [], 0
        for key in keys:
            zi, source = members[key]
            c = zi.compress_size + 3 * zi.file_size + 1024
            if batch and cost + c > batch_bytes:
                uploaded += Z.decode_members(decoder, batch, part_done)
                batch, cost = [], 0
            batch.append((key, zi, source))
            cost += c
        if batch:
            uploaded += Z.decode_members(decoder, batch, part_done)
        return uploaded
    return decode


def check_entries(entries, decode, parser, mount="/var/task", arch="x86_64", provided=DEFAULT_PROVIDED,
                  max_versions=None, ld_library_path=LAMBDA_LD_LIBRARY_PATH, *, symbols=False, interpreter=(),
                  runtime_libs=(), resolver=None, python_names=True, python=None):
    """The check over the entries of a zip: entries [(key, name, link)] (an opaque hashable key, the entry's name, a
    symlink's target or None), in the zip's order.  decode(keys, consume) puts the regular files of a round on the
    device: it calls consume(part, refs) once or more, part a list of the keys and refs their (device address, size),
    valid until consume returns, and returns the bytes it uploaded.  The report has no inflate_ms: the caller knows
    what its decode step cost."""
    if (symbols or python) and resolver is None:
        raise ValueError("symbols=True and python need a resolver")
    ceilings = _ceilings(arch, max_versions)
    python_version(python)
    sym_ids = {}
    tree = _Tree(entries, mount)
    path_of = {}
    for p, key in tree.files.items():
        path_of.setdefault(key, p)
    roots = [(p, key) for p, key in sorted(tree.files.items())
             if tree.names[key].rsplit("/", 1)[-1].endswith(Z.SO_SUFFIX)]  # Z.selected_for_strip of a regular file
    objs, rounds, uploaded = {}, 0, 0
    model = _Model(tree, objs, arch, provided, ld_library_path)

    def consume(keys, refs):
        if symbols or python:  # before parse(), which frees the uploads
            for key, got in zip(keys, resolver.index(refs)):
                sym_ids[key] = got
        for key, (status, machine, records) in zip(keys, parser.parse(refs)):
            objs[key] = _Obj(tree.names[key], status, machine, records)

    todo = [key for _, key in roots]
    while todo:
        rounds += 1
        uploaded += decode(todo, consume)
        seen, todo = set(), []
        for p, key in roots:
            for k in model.closure(p, key)[2]:
                if k not in objs and k not in seen:
                    seen.add(k)
                    todo.append(k)
    report = _report(tree, roots, objs, model, path_of, arch, ceilings)
    report["stats"] = {"members": len(entries), "roots": len(roots), "objects": len(objs), "rounds": rounds,
                       "bytes_up": uploaded + parser.uploaded, "bytes_down": parser.downloaded,
                       "parse_ms": parser.stats().get("kernel_ms", 0.0)}
    counted = (0, 0)
    if symbols:
        _Symbols(tree, roots, objs, model, path_of, sym_ids, parser, resolver, provided, interpreter, runtime_libs,
                 python_names).check(report)
        counted = (resolver.uploaded, resolver.downloaded)
    if python:
        _imports(report, tree, roots, objs, model, path_of, sym_ids, resolver, python, arch, counted)
    return report


def check_with(zip_path, decoder, parser, mount="/var/task", arch="x86_64", provided=DEFAULT_PROVIDED,
               max_versions=None, ld_library_path=LAMBDA_LD_LIBRARY_PATH, batch_bytes=BATCH_BYTES, *, symbols=False,
               interpreter=(), runtime_libs=(), resolver=None, python_names=True, python=None):
    """check_zip with the engines given (GpuUnzipDecoder, GpuElfParser and, with symbols=True or python,
    GpuSymbolResolver, or stand-ins with the same interfaces).  python_names=False turns off the rule that counts an
    unresolved Py* / _Py* name as the interpreter's when no interpreter is given."""
    if (symbols or python) and resolver is None:
        raise ValueError("symbols=True and python need a resolver")
    _ceilings(arch, max_versions)
    python_version(python)
    with zipfile.ZipFile(zip_path) as zf, open(zip_path, "rb") as src:
        src.seek(0, os.SEEK_END)
        source = (zf, src, src.tell())
        infos = zf.infolist()
        entries = [(i, zi.filename, zf.read(zi).decode("utf-8", "surrogateescape")
                    if not zi.is_dir() and (zi.external_attr >> 16) & 0o170000 == stat.S_IFLNK else None)
                   for i, zi in enumerate(infos)]
        decode = member_decoder(decoder, parser, {i: (zi, source) for i, zi in enumerate(infos)}, batch_bytes)
        report = check_entries(entries, decode, parser, mount, arch, provided, max_versions, ld_library_path,
                               symbols=symbols, interpreter=interpreter, runtime_libs=runtime_libs, resolver=resolver,
                               python_names=python_names, python=python)
    report["stats"]["inflate_ms"] = decoder.stats().get("kernel_ms", 0.0)
    return report


def _report(tree, roots, objs, model, path_of, arch, ceilings):
    problems, notes, seen = [], [], set()
    highest, provided_used = {}, {}

    def problem(obj, kind, detail, weak=False):
        key = (obj, kind, detail)
        if key not in seen:
            seen.add(key)
            (notes if weak else problems).append({"object": obj, "kind": kind, "detail": detail})

    objects, closures, resolved = {}, {}, {}
    for key, o in objs.items():
        p = path_of[key]
        objects[p] = {"member": o.member, "status": STATUS_NAMES.get(o.status, str(o.status)),
                      "machine": o.machine, "soname": o.soname, "rpath": o.rpath, "runpath": o.runpath, "needed": None,
                      "version_needs": [{"file": f, "version": v, "weak": w} for f, v, w in o.verneed],
                      "version_defs": sorted(o.verdef)}
    for root_path, root_key in roots:
        loaded, resolutions, _ = model.closure(root_path, root_key)
        closures[root_path] = [path_of[key] for _, key in loaded]
        by_name, filled = {}, set()  # names in this closure -> (how, path)
        resolved[root_path] = [{"object": path_of[lkey], "name": name, "how": how,
                                "path": found and posixpath.normpath(found)} for _, lkey, name, how, found in resolutions]
        for loader_path, lkey, name, how, found in resolutions:
            by_name.setdefault(name, (how, found))
            loader_path = posixpath.normpath(loader_path)
            o = objects[path_of[lkey]]
            if o["needed"] is None:
                o["needed"] = []
                filled.add(lkey)
            if lkey in filled:
                o["needed"].append({"name": name, "how": how, "path": found and posixpath.normpath(found)})
            if how == "missing":
                problem(loader_path, "missing", "%s: not in the zip, the search path or the runtime" % name)
            elif how == "provided":
                provided_used.setdefault(name, set()).add(loader_path)
        filled = set()
        for p, key in loaded:
            p = posixpath.normpath(p)
            o = objs[key]
            if o.status != N.ELF_OK:
                problem(p, "unloadable", "%s: %s" % (o.member, STATUS_NAMES.get(o.status, o.status)))
                continue
            if o.machine != MACHINES[arch]:
                problem(p, "arch", "e_machine %d, not %s (%d)" % (o.machine, arch, MACHINES[arch]))
            for f, v, weak in o.verneed:
                how, found = by_name.get(f, (None, None))
                if how == "provided":
                    m = _VERSION.match(v)
                    if m:
                        prefix, key = m.group(1), _version_key(m.group(2))
                        if prefix not in highest or key > _version_key(highest[prefix]):
                            highest[prefix] = m.group(2)
                        if prefix in ceilings and key > ceilings[prefix]:
                            problem(p, "version", "%s from %s is newer than the runtime's %s_%s"
                                    % (v, f, prefix, ".".join(map(str, ceilings[prefix]))), weak)
                elif found is not None:
                    t = objs.get(tree.lookup(found))
                    if t is not None and t.status == N.ELF_OK and v not in t.verdef:
                        if not t.verdef:
                            problem(p, "version", "%s: %s has no version information" % (v, f), True)
                        else:
                            problem(p, "version", "%s not defined by %s" % (v, f), weak)
    return {"arch": arch, "mount": tree.mount, "objects": objects, "closures": closures, "resolved": resolved,
            "problems": problems,
            "notes": notes, "max_versions": dict(sorted(highest.items())),
            "provided_used": {k: sorted(v) for k, v in sorted(provided_used.items())}}


class _Symbols:
    """The symbol check of check_with(symbols=True) over the parsed zip: the scope of each root, the lookups of the
    references of every object in its closure (by the resolver), and the classes and problems of what is left."""

    def __init__(self, tree, roots, objs, model, path_of, sym_ids, parser, resolver, provided, interpreter,
                 runtime_libs, python_names):
        self.tree, self.roots, self.objs, self.model, self.path_of = tree, roots, objs, model, path_of
        self.sym_ids, self.parser, self.resolver = sym_ids, parser, resolver
        self.provided, self.interpreter, self.runtime_libs = frozenset(provided), list(interpreter), list(runtime_libs)
        self.python_names = python_names
        self.host = {}  # real path of an interpreter file or runtime library -> (class, (id, status, refs), _Obj, path)

    def _load(self, path, cls):
        real = os.path.realpath(path)
        if real not in self.host:
            with open(real, "rb") as f:
                data = f.read()
            ref = self.parser.upload(data)
            sym = self.resolver.index([ref])[0]
            status, machine, records = self.parser.parse([ref])[0]
            self.host[real] = (cls, sym, _Obj(None, status, machine, records), path)
        return real

    def _runtime(self, name):
        """the real path of `name` in runtime_libs, loaded, or None"""
        for d in self.runtime_libs:
            p = os.path.join(d, name)
            if os.path.isfile(p):
                return self._load(p, CLASS_RUNTIME)
        return None

    def _host_needs(self, real):
        """the nodes of a host object's DT_NEEDED, found in its DT_RPATH / DT_RUNPATH ($ORIGIN expanded), then in
        runtime_libs; a name found nowhere is a provided node when it is in `provided`, else left out"""
        cls, _, o, path = self.host[real]
        dirs = []
        for rp in (o.rpath, o.runpath):
            for d in rp.split(":") if rp else ():
                dirs.append(d.replace("${ORIGIN}", os.path.dirname(path)).replace("$ORIGIN", os.path.dirname(path)))
        out = []
        for name in o.needed:
            node = next((("host", self._load(os.path.join(d, name), cls)) for d in dirs
                         if os.path.isfile(os.path.join(d, name))), None)
            if node is None:
                r = self._runtime(name)
                node = ("host", r) if r else ("provided", name) if name in self.provided else None
            if node is not None:
                out.append(node)
        return out

    def _bfs(self, order, needs):
        seen, q = set(order), 0
        while q < len(order):
            for node in needs(order[q]):
                if node not in seen:
                    seen.add(node)
                    order.append(node)
            q += 1
        return order

    def _local(self, root_key, resolutions):
        """the root's search list: the closure's breadth-first order with the provided libraries at their places"""
        by_loader = {}
        for _, lkey, name, how, found in resolutions:
            by_loader.setdefault(lkey, []).append((name, how, found))

        def needs(node):
            kind, key = node
            if kind == "host":
                return self._host_needs(key)
            out = []
            for name, how, found in by_loader.get(key, []) if kind == "zip" else ():
                if how == "provided":
                    r = self._runtime(name)
                    out.append(("host", r) if r else ("provided", name))
                elif how != "missing":
                    out.append(("zip", self.tree.lookup(found)))
            return out
        return self._bfs([("zip", root_key)], needs)

    def check(self, report):
        up0, down0 = self.parser.uploaded, self.parser.downloaded
        problems, notes = report["problems"], report["notes"]
        seen = {(p["object"], p["kind"], p["detail"]) for p in problems + notes}

        def problem(obj, kind, detail, weak=False):
            if (obj, kind, detail) not in seen:
                seen.add((obj, kind, detail))
                (notes if weak else problems).append({"object": obj, "kind": kind, "detail": detail})

        glob = self._bfs([("host", self._load(f, CLASS_INTERPRETER)) for f in self.interpreter],
                         lambda node: self._host_needs(node[1]) if node[0] == "host" else [])
        jobs, flat, scopes, meta, first, symbols, skipped = [], [], {}, [], {}, {}, 0
        for root_path, root_key in self.roots:
            loaded, resolutions, _ = self.model.closure(root_path, root_key)
            if any(r[3] == "missing" for r in resolutions) or any(self.objs[k].status != N.ELF_OK for _, k in loaded):
                skipped += 1
                continue
            order, ids, opaque = [], [], []
            for node in glob + self._local(root_key, resolutions):
                if node in order:
                    continue
                order.append(node)
                kind, key = node
                if kind == "provided":
                    opaque.append(key)
                else:
                    ids.append(self.sym_ids[key][0] if kind == "zip" else self.host[key][1][0])
            skey = (tuple(ids), tuple(opaque))
            if skey not in scopes:
                scopes[skey] = len(flat)
                flat += ids
            root = posixpath.normpath(root_path)
            for p, key in loaded:
                p = posixpath.normpath(p)
                rid, status, nrefs = self.sym_ids[key]
                if status != N.SYM_OK:
                    problem(p, "symbol", "symbol tables %s: not checked" % STATUS_NAMES.get(status, status),
                            status == N.SYM_UNSUPPORTED)
                    continue
                symbols.setdefault(p, {"references": nrefs, "in_zip": 0, "runtime": 0, "trusted": 0, "interpreter": 0,
                                       "unverified": 0})
                if nrefs and (rid, skey) not in first:
                    first[(rid, skey)] = len(jobs)
                    jobs.append((rid, scopes[skey], len(ids)))
                    meta.append((p, root, opaque))
        n_ids = 1 + max([s[0] for s in self.sym_ids.values()] + [h[1][0] for h in self.host.values()] + [0])
        classes = [CLASS_IN_ZIP] * n_ids
        for cls, sym, _, _ in self.host.values():
            classes[sym[0]] = cls
        counts, misses = self.resolver.resolve(jobs, flat, classes)
        per = [{"in_zip": c[0], "runtime": c[1], "interpreter": c[2], "trusted": 0, "unverified": 0} for c in counts]
        reported = set()  # (object, symbol): one problem or note each, under the first root that met it
        for (j, _), (name, ver, file) in zip(misses, self.resolver.names(jobs, misses)):
            p, root, opaque = meta[j]
            label = name + ("@" + ver if ver else "")
            first_report = (p, label) not in reported
            reported.add((p, label))
            if not self.interpreter and self.python_names and name.startswith(("Py", "_Py")):
                per[j]["interpreter"] += 1
            elif ver and file in self.provided and self._runtime(file) is None:
                per[j]["trusted"] += 1
            elif not ver and opaque:  # glibc binds it to a definition at versym index 2 too (DESIGN.md section 9.9)
                per[j]["unverified"] += 1
                if first_report:
                    problem(p, "symbol", "%s: not found; unverified: %s may define it" % (label, ", ".join(opaque)), True)
            elif first_report:
                problem(p, "symbol", "%s: no definition in the load scope of %s" % (label, root))
        seen_obj = set()
        for j, (p, _, _) in enumerate(meta):
            if p not in seen_obj:
                seen_obj.add(p)
                symbols[p].update(per[j])
        # a version need on a provided library read from runtime_libs: its Verdefs must have it
        for key, o in self.objs.items():
            if o.status != N.ELF_OK:
                continue
            for f, v, weak in o.verneed:
                real = self._runtime(f) if f in self.provided else None
                if real is not None and self.host[real][2].status == N.ELF_OK and v not in self.host[real][2].verdef:
                    problem(posixpath.normpath(self.path_of[key]), "version", "%s not defined by %s" % (v, f), weak)
        st, rs = report["stats"], self.resolver.stats()
        refs_of = {i: n for i, _, n in self.sym_ids.values()}
        report["symbols"] = dict(sorted(symbols.items()))
        st["bytes_up"] += self.parser.uploaded - up0 + self.resolver.uploaded
        st["bytes_down"] += self.parser.downloaded - down0 + self.resolver.downloaded
        st.update({"symbols_ms": rs["index_ms"] + rs["refs_ms"] + rs["resolve_ms"], "symbols_index_ms": rs["index_ms"],
                   "symbols_refs_ms": rs["refs_ms"], "symbols_resolve_ms": rs["resolve_ms"],
                   "references": sum(refs_of[j[0]] for j in jobs), "lookups": rs["lookups"],
                   "symbols_skipped": skipped})


def python_version(python):
    """python, refused unless None or one of PYTHON_VERSIONS ("3.8" .. "3.14"; free-threaded builds are not)"""
    if python is not None and python not in PYTHON_VERSIONS:
        raise ValueError("python=%r: expected one of %s" % (python, ", ".join(PYTHON_VERSIONS)))
    return python


def export_name(module):
    """the PyInit_* name CPython looks up for the extension module `module` (importdl.c get_encoded_name and
    dynload_shlib.c: the last dotted component, punycode with '-' as '_' and the PyInitU prefix when it is not ASCII,
    cut to 200 bytes)"""
    short = module.rsplit(".", 1)[-1]
    try:
        prefix, enc = b"PyInit", short.encode("ascii")
    except UnicodeEncodeError:
        prefix, enc = b"PyInitU", short.encode("punycode")
    return prefix + b"_" + enc.replace(b"-", b"_")[:200]


class _Finder:
    """CPython's PathFinder with FileFinders of the target's loaders (importlib._bootstrap_external,
    _get_supported_file_loaders) over the tree: the extension suffixes, then .py, then .pyc"""

    def __init__(self, tree, version, arch):
        self.tree = tree
        self.ext = [".cpython-3%s-%s.so" % (version.split(".")[1], TRIPLETS[arch]), ".abi3.so", ".so"]
        self.suffixes = self.ext + [".py", ".pyc"]
        self.path = [p.format(version=version) for p in LAMBDA_PYTHON_PATH]
        m = tree.mount
        self.entries = [p for p in self.path if m == "/" or p == m or p.startswith(m + "/")]
        self._specs = {}

    def _in_dir(self, d, tail):
        """FileFinder(d).find_spec(tail): (origin, None) for a module, (origin, [dir]) for a regular package,
        (None, [dir]) for a namespace portion, or None"""
        cd = self.tree.directory(d)
        if cd is None:
            return None
        names, base, namespace = self.tree.children(cd), d + "/" + tail, False
        if tail in names:
            for suffix in self.suffixes:
                if self.tree.lookup(base + "/__init__" + suffix) is not None:
                    return base + "/__init__" + suffix, [base]
            namespace = self.tree.directory(base) is not None
        for suffix in self.suffixes:
            if tail + suffix in names and self.tree.lookup(d + "/" + tail + suffix) is not None:
                return d + "/" + tail + suffix, None
        return (None, [base]) if namespace else None

    def find(self, module):
        """(origin or None, __path__ or None) of the dotted name `module` as `import` finds it, or None"""
        if module not in self._specs:
            parent, _, tail = module.rpartition(".")
            search = self.entries
            if parent:
                spec = self.find(parent)
                search = spec[1] if spec else None
            found, portions = None, []
            for d in search or ():
                got = self._in_dir(d, tail)
                if got and got[0] is not None:
                    found = got
                    break
                portions += got[1] if got else []
            self._specs[module] = found or ((None, portions) if portions else None)
        return self._specs[module]

    def name(self, path):
        """(dotted module name, suffix, tag) of the file `path` under a path entry: tag None when its suffix is one of
        the target's, else the other Python's tag; None when no importable name fits it"""
        for e in self.entries:
            if not path.startswith(e + "/"):
                continue
            parts = path[len(e) + 1:].split("/")
            base, tag = parts.pop(), None
            suffix = next((x for x in self.ext if base.endswith(x) and base[:-len(x)].isidentifier()), None)
            if suffix is not None:
                stem = base[:-len(suffix)]
            else:
                m = _PY_TAG.match(base)
                if not m:
                    return None
                stem, tag, suffix = m.group(1), m.group(2), "." + m.group(2) + ".so"
            parts += [] if stem == "__init__" else [stem]
            if parts and all(x.isidentifier() for x in parts):
                return ".".join(parts), suffix, tag
        return None


def _imports(report, tree, roots, objs, model, path_of, sym_ids, resolver, version, arch, counted):
    """The import check of check_entries(python=version): report["python"], problems and notes of kind "python" and
    the stats modules, python_skipped, find_queries and find_ms.  counted: the resolver's (uploaded, downloaded)
    bytes already in the report's stats."""
    finder = _Finder(tree, version, arch)
    problems, notes = report["problems"], report["notes"]
    seen = {(p["object"], p["kind"], p["detail"]) for p in problems + notes}

    def problem(obj, detail, weak=False):
        if (obj, "python", detail) not in seen:
            seen.add((obj, "python", detail))
            (notes if weak else problems).append({"object": obj, "kind": "python", "detail": detail})

    def what(spec):
        if spec is None:
            return "no module"
        return spec[0] if spec[0] is not None else "the namespace package " + ":".join(spec[1])

    path_by_id = {sid[0]: posixpath.normpath(path_of[k]) for k, sid in sym_ids.items()}
    modules, queries, qmeta, flat, scopes, skipped = {}, [], [], [], {}, 0
    for root_path, key in roots:
        p = posixpath.normpath(root_path)
        if not any(p.startswith(e + "/") for e in finder.entries):
            continue
        got = finder.name(p)
        rec = {"module": None, "class": "library", "export": None, "defined_by": None, "status": None}
        modules[p] = rec
        if got is None:
            continue
        module, suffix, tag = got
        spec = finder.find(module)
        rec["module"] = module
        if tag is not None:
            rec["class"] = "other python"
            if spec is None:
                problem(p, "%s: built only for %s; Python %s finds no module %s" % (module, tag, version, module))
            else:
                problem(p, "%s: built for %s, which Python %s does not load; it imports %s"
                        % (module, tag, version, what(spec)), True)
            continue
        if spec is None or spec[0] is None or tree.lookup(spec[0]) != key:
            rec["class"] = "shadowed"
            problem(p, "%s: never loaded: Python %s imports %s" % (module, version, what(spec)), True)
            continue
        rec["class"], rec["export"] = "module", export_name(module).decode("ascii")
        loaded, resolutions, _ = model.closure(root_path, key)
        if any(r[3] == "missing" for r in resolutions) or any(objs[k].status != N.ELF_OK for _, k in loaded) or \
                sym_ids[key][1] != N.SYM_OK:
            rec["status"] = "not checked"
            skipped += 1
            continue
        ids = tuple(sym_ids[k][0] for _, k in loaded)  # provided libraries are not read: they define no PyInit_*
        if ids not in scopes:
            scopes[ids] = len(flat)
            flat += ids
        queries.append((scopes[ids], len(ids), export_name(module)))
        qmeta.append((p, suffix))
    ms0 = resolver.stats().get("find_ms", 0.0)
    for (p, suffix), (obj, _, _, _, _) in zip(qmeta, resolver.find(queries, flat)):
        rec = modules[p]
        if obj is not None:
            rec["status"], rec["defined_by"] = "ok", path_by_id[obj]
        elif suffix == ".so":  # a bare .so without the export: a library that happens to be importable by name
            rec.update({"module": None, "class": "library", "export": None})
        else:
            rec["status"] = "not exported"
            problem(p, '%s not exported: the import fails with "dynamic module does not define module export function"'
                    % rec["export"])
    st = report["stats"]
    st["bytes_up"] += resolver.uploaded - counted[0]
    st["bytes_down"] += resolver.downloaded - counted[1]
    st.update({"modules": sum(1 for r in modules.values() if r["class"] == "module"), "python_skipped": skipped,
               "find_queries": len(queries), "find_ms": resolver.stats().get("find_ms", 0.0) - ms0})
    report["python"] = {"version": version, "path": finder.path, "modules": dict(sorted(modules.items()))}


def check_zip(zip_path, mount="/var/task", arch="x86_64", provided=DEFAULT_PROVIDED, max_versions=None,
              ld_library_path=LAMBDA_LD_LIBRARY_PATH, ctx=None, batch_bytes=BATCH_BYTES, *, symbols=False,
              interpreter=(), runtime_libs=(), python=None):
    """Check that the shared objects of `zip_path`, unpacked at `mount`, will load on Lambda (see the module docstring
    for the search it restates).  Returns a plain dict:

    * objects: {mounted path: member, status ("ok", "not ELF", "unsupported", "static", "malformed"), machine, soname,
      rpath, runpath, needed [{name, how ("rpath", "ld_library_path", "runpath", "path", "loaded", "provided",
      "missing"), path}] as the first root that loaded it resolved them, version_needs, version_defs};
    * closures: {root: the members its dlopen loads (as keys of objects), in load order}; resolved: {root: every
      need met in that load, [{object, name, how, path}] in the loader's order};
    * problems [{object, kind, detail}]: kind "missing" (a DT_NEEDED resolved nowhere), "arch" (e_machine is not
      `arch`'s: x86_64 62, arm64 183), "version" (a version need not defined by the member it resolved to, or above
      the `max_versions` ceiling of its prefix on a provided library, such as {"GLIBC": "2.26"}), "unloadable" (a
      loaded object that is not an ELF64 little-endian shared object with a dynamic section); weak version needs and
      needs on members without version information go to notes instead;
    * max_versions: the highest version needed of each prefix (GLIBC, GLIBCXX, CXXABI, GCC ...) on provided
      libraries; provided_used: {soname: the objects whose need the `provided` list satisfied};
    * stats: members, roots, objects (parsed), rounds, bytes_up, bytes_down, inflate_ms and parse_ms (CUDA events).

    symbols=True also checks that every symbol the objects' relocations look up has a definition in the scope of a
    `dlopen(root, RTLD_NOW | RTLD_LOCAL)` from the interpreter (DESIGN.md section 9.9): the exported definitions of
    the `interpreter` files (such as sys.executable) and their DT_NEEDED closure, then the root's closure in load
    order.  `runtime_libs` are host directories holding the `provided` libraries; one found there takes its place in
    the scope with its own definitions.  The report gains problems of kind "symbol" (NAME[@VERSION]: no definition in
    the load scope of ROOT), notes of kind "symbol" (an unversioned name that only a provided library not read could
    define), "version" problems against the Verdefs of the runtime_libs copies, symbols {object: {references, in_zip,
    runtime, trusted, interpreter, unverified}} under the first root that checked it, and stats symbols_ms (index,
    refs and resolve kernels, CUDA events; also split as symbols_index_ms, symbols_refs_ms, symbols_resolve_ms),
    references, lookups and symbols_skipped (roots with a missing need or an unloadable object, not checked).

    python="3.N" (3.8 .. 3.14) also checks that the extension modules will import on that Python (DESIGN.md section
    9.11): CPython's finder restated on LAMBDA_PYTHON_PATH's entries under `mount`, with the target's suffixes
    (.cpython-3N-<arch triplet>.so, .abi3.so, .so, then .py, .pyc), and each module's PyInit_<name> looked up in its
    load scope as dlsym looks it up.  The report gains python {version, path (the sys.path modelled), modules {mounted
    path of every *.so under a path entry: module (dotted name), class ("module", "shadowed", "other python",
    "library"), export, defined_by, status ("ok", "not exported", "not checked"; modules only)}}, problems of kind
    "python" (a build only for another Python whose name the finder does not find; a module without its PyInit_*),
    notes of kind "python" (a shadowed file; a build for another Python beside one that loads) and stats modules,
    python_skipped (modules with a missing need or an unloadable object, not looked up), find_queries and find_ms.

    Members are inflated by the GPU zip reader and parsed on the GPU (lb2_elf_deps) where they lie; only the records
    and their strings come back.  There is no CPU path: without a GPU this raises."""
    from .tarball import _default_context
    own = False
    if ctx is None:
        ctx, own = _default_context()
    python_version(python)
    try:
        with Z.GpuUnzipDecoder(ctx) as dec, GpuElfParser(ctx) as parser:
            if not symbols and not python:
                return check_with(zip_path, dec, parser, mount, arch, provided, max_versions, ld_library_path, batch_bytes)
            with GpuSymbolResolver(ctx) as resolver:
                return check_with(zip_path, dec, parser, mount, arch, provided, max_versions, ld_library_path,
                                  batch_bytes, symbols=symbols, interpreter=interpreter, runtime_libs=runtime_libs,
                                  resolver=resolver, python=python)
    finally:
        if own:
            ctx.close()


def summary(report):
    st = report["stats"]
    lines = ["%d shared objects checked (%d roots, %d rounds) under %s for %s: %d problem(s)"
             % (st["objects"], st["roots"], st["rounds"], report["mount"], report["arch"], len(report["problems"]))]
    if report["max_versions"]:
        lines.append("highest versions needed: " + ", ".join("%s_%s" % kv for kv in report["max_versions"].items()))
    if report["provided_used"]:
        lines.append("satisfied by the runtime list: " + ", ".join(report["provided_used"]))
    if "symbols" in report:
        lines.append("symbols: %d references, %d lookups, %d root(s) not checked"
                     % (st["references"], st["lookups"], st["symbols_skipped"]))
    if "python" in report:
        lines.append("python %s: %d extension modules, %d not checked, %d PyInit lookups"
                     % (report["python"]["version"], st["modules"], st["python_skipped"], st["find_queries"]))
    for p in report["problems"]:
        lines.append("problem: %s: %s: %s" % (p["object"], p["kind"], p["detail"]))
    for p in report["notes"]:
        lines.append("note: %s: %s: %s" % (p["object"], p["kind"], p["detail"]))
    return "\n".join(lines)


def _ceiling(text):
    m = _VERSION.match(text)
    if not m:
        raise ValueError("--max-version %r: expected PREFIX_VERSION such as GLIBC_2.26" % text)
    return m.group(1), m.group(2)


def add_check_arguments(ap):
    """the check's options on the ArgumentParser ap; returns their destinations (check_kwargs reads them)"""
    ap.add_argument("--mount", default="/var/task", help="where the zip is unpacked: /var/task (function) or /opt (layer)")
    ap.add_argument("--arch", choices=sorted(MACHINES), default="x86_64")
    ap.add_argument("--provided", action="append", metavar="NAME",
                    help="a soname the runtime supplies (repeatable; replaces the default list)")
    ap.add_argument("--max-version", action="append", default=[], metavar="PREFIX_VERSION",
                    help="the runtime's highest version of a prefix, such as GLIBC_2.26 (repeatable)")
    ap.add_argument("--ld-library-path", default=LAMBDA_LD_LIBRARY_PATH)
    ap.add_argument("--symbols", action="store_true", help="also check the symbols each object binds when it loads")
    ap.add_argument("--interpreter", action="append", default=[], metavar="FILE",
                    help="with --symbols: an ELF file heading the global scope, such as the python executable (repeatable)")
    ap.add_argument("--runtime-lib", action="append", default=[], metavar="DIR",
                    help="with --symbols: a directory holding the runtime's provided libraries (repeatable)")
    ap.add_argument("--python", metavar="3.N", help="also check that the extension modules import on this Python "
                                                    "(%s .. %s)" % (PYTHON_VERSIONS[0], PYTHON_VERSIONS[-1]))
    return ("mount", "arch", "provided", "max_version", "ld_library_path", "symbols", "interpreter", "runtime_lib",
            "python")


def check_kwargs(args):
    """check_zip's keyword arguments from the options add_check_arguments defined; ValueError for a --max-version
    that is not PREFIX_VERSION or a --python that is not one of PYTHON_VERSIONS"""
    return dict(mount=args.mount, arch=args.arch,
                provided=DEFAULT_PROVIDED if args.provided is None else frozenset(args.provided),
                max_versions=dict(_ceiling(t) for t in args.max_version), ld_library_path=args.ld_library_path,
                **({"symbols": True, "interpreter": args.interpreter, "runtime_libs": args.runtime_lib}
                   if args.symbols else {}),
                **({"python": python_version(args.python)} if args.python is not None else {}))


def main(argv=None, check=check_zip):
    """exit status 0: no problem; 1: problems; 2: a refused input or a usage error"""
    import argparse
    ap = argparse.ArgumentParser(prog="python -m lambdipy_b200.deps",
                                 description="check that the shared objects of a Lambda zip will load there")
    ap.add_argument("zip")
    add_check_arguments(ap)
    ap.add_argument("--json", action="store_true", help="print the whole report as JSON")
    args = ap.parse_args(argv)
    try:
        report = check(args.zip, **check_kwargs(args))
    except (OSError, ValueError, zipfile.BadZipFile) as e:
        print("error: %s" % e, file=sys.stderr)
        return 2
    print(json.dumps(report, indent=1, sort_keys=True) if args.json else summary(report))
    return 1 if report["problems"] else 0


if __name__ == "__main__":
    sys.exit(main())
