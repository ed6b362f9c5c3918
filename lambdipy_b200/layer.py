"""The Lambda zip of package tarballs, converted on the GPU without unpacking them.

Prebuilt packages arrive as .tar.gz release assets (tarball.prepare_tarfile, create_compressed_tarball) and Lambda
takes a zip.  Building a layer from them used to take four passes over the disk: extract each asset, run the strip line
on the tree, walk and read the tree again for zip_tree, write the zip.  zip_tarballs chains the engines that already
exist in device memory instead:

    1. every source is uploaded once and inflated into one device arena (tarball.GpuTarReader.read_many);
    2. one warp walks each tar stream's headers (lb2_tar_index) so that tarfile lists its members from one download;
    3. on the host the member lists are merged as consecutive extractall()s would merge them, the `*.so` files are
       selected as `find -name "*.so" | xargs strip` would find them, and the entries are listed as make_archive
       would walk the tree;
    4. the selected files are stripped where they lie, in one batch (zipfile_gpu.GpuStripper);
    5. every file entry is deflated straight from the arena or the stripped arena (lb2_zip_submit_device), and the
       container is written by zipfile_gpu's writer.

Only compressed bytes cross the bus: the sources going up, the index and the DEFLATE bodies coming down, and the files
the host `strip` fallback handles.

    zip_tarballs(srcs, dst, prefix="")
    python -m lambdipy_b200.layer DST SRC [SRC ...] [--prefix python/] [--level 9] [--seek-table]

zip_build adds wheels to the same chain: pip's `--target` install and the build script's clean-up lines are restated
on the merged tree, the wheels' shared objects are inflated on the GPU next to the tarballs' files, and every other
wheel member's DEFLATE body is copied into the zip as it is.

    zip_build(dst, tarballs=(), wheels=(), prefix="", keep_tests=())
    python -m lambdipy_b200.layer DST [SRC ...] --wheel WHL [--wheel WHL ...] [--keep-tests NAME] [--clean]

Both writers take check={...} (--check): deps.check_zip's check of the zip, run on the stripped objects where they lie
on the device before the zip is written; a problem raises deps.CheckFailed and writes nothing (DESIGN.md section 9.10).
"""
import contextlib
import ctypes as C
import email.parser
import importlib.metadata
import os
import posixpath
import re
import stat
import struct
import sys
import tempfile
import time
import zipfile
import zlib

from . import _native as N
from . import deps as D
from . import seek_table as ST
from . import tarball as T
from . import zipfile_gpu as Z

PIECE_BYTES = Z.PIECE_BYTES


class _Dir:
    """a directory of the merged tree; mode / mtime None: made by makedirs, with no member of its own"""

    def __init__(self):
        self.mode = self.mtime = None


class _File:
    """a regular file of the merged tree (an inode: hard links share it): the source and member holding its data,
    the mode and mtime tarfile applied to it last, and how many names it has"""

    def __init__(self):
        self.src, self.member, self.mode, self.mtime, self.links = None, None, 0, 0, 1

    def position(self):
        """where the file's data lies among the sources: the order the stripper takes it in"""
        return self.src, self.member.offset_data

    def label(self):
        return self.member.name


class _Link:
    def __init__(self, target):
        self.target = target


class _Special:
    """a FIFO or device node: os.path.isfile is False, so make_archive writes no entry"""


def check_prefix(prefix):
    if prefix and (not prefix.endswith("/") or prefix.startswith("/") or
                   any(c in ("", ".", "..") for c in prefix[:-1].split("/"))):
        raise ValueError("prefix %r: empty, or relative path components ending in '/' (e.g. 'python/')" % prefix)


def _path(prefix, name):
    """the path under the zip's root that extracting `name` under `prefix` writes to ("" is the root)"""
    n = posixpath.normpath(name) if name else "."
    if T._leaves(n):
        raise ValueError("member %r leaves the directory it is extracted to" % name)
    return prefix[:-1] if n == "." else prefix + n


def lookup(nodes, path):
    """The node a path of the merged tree ends at, symlinks followed (a link target joined to the link's directory and
    normalised, as select_members resolves it), or None: dangling, through a non-directory, leaving the tree or more
    than 40 links."""
    parts, i, cur, hops = path.split("/") if path else [], 0, "", T._SYMLINK_HOPS
    while i < len(parts):
        nxt = parts[i] if not cur else cur + "/" + parts[i]
        node = nodes.get(nxt)
        if isinstance(node, _Link):
            hops -= 1
            if hops < 0 or node.target.startswith("/"):
                return None
            path = posixpath.normpath(posixpath.join(posixpath.dirname(nxt), node.target, *parts[i + 1:]))
            if T._leaves(path):
                return None
            parts, i, cur = [] if path == "." else path.split("/"), 0, ""
            continue
        if node is None or (i + 1 < len(parts) and not isinstance(node, _Dir)):
            return None
        cur, i = nxt, i + 1
    return nodes.get(cur)


def merge(listings, prefix=""):
    """The tree that `extractall(tree / prefix, filter="fully_trusted")` of each source in order leaves, from the
    sources' member lists: {path: _Dir | _File | _Link | _Special}, the root "" included.

    A later member replaces an earlier one of the same name only directory onto directory and regular file onto
    regular file (extractall rewrites the file in place); any other collision, replacing a file a hard link shares,
    a member below a symlink or a file, a name leaving the tree, a hard link not ending at a regular file, a sparse
    member and an unknown member type raise ValueError."""
    check_prefix(prefix)
    nodes = {"": _Dir()}
    for k in range(prefix.count("/")):
        nodes["/".join(prefix.split("/")[:k + 1])] = _Dir()
    for src, members in enumerate(listings):
        for m in members:
            name = _path(prefix, m.name)
            if not name:
                if not m.isdir():
                    raise ValueError("member %r is the directory it is extracted to" % m.name)
                continue
            parts = name.split("/")
            for k in range(1, len(parts)):
                up = "/".join(parts[:k])
                node = nodes.setdefault(up, _Dir())
                if not isinstance(node, _Dir):
                    raise ValueError("member %r: %r is not a directory of the tree" % (m.name, up))
            old = nodes.get(name)

            def collision(why):
                return ValueError("member %r of source %d: %s" % (m.name, src, why))
            if m.issparse():
                raise ValueError("member %r is sparse: its data is not in the tar stream" % m.name)
            if m.isdir():
                if old is not None and not isinstance(old, _Dir):
                    raise collision("a directory onto a non-directory")
                node = old or _Dir()
            elif m.isreg():
                if old is not None and not isinstance(old, _File):
                    raise collision("a file onto a directory, link or special file")
                if old is not None and old.links > 1:
                    raise collision("replaces a file that a hard link shares")
                node = old or _File()
                node.src, node.member = src, m
            elif old is not None:
                raise collision("a link or special file onto an existing entry")
            elif m.issym():
                node = _Link(m.linkname)
            elif m.islnk():
                node = lookup(nodes, _path(prefix, m.linkname))
                if not isinstance(node, _File):
                    raise ValueError("hard link %r: %r is not a regular file of the tree" % (m.name, m.linkname))
                node.links += 1
            elif m.isfifo() or m.ischr() or m.isblk():
                node = _Special()
            else:
                raise ValueError("member %r has an unsupported type %r" % (m.name, m.type))
            if not m.issym():
                node.mode, node.mtime = m.mode, m.mtime
            nodes[name] = node
    return nodes


def walk(nodes):
    """([(path, node)] of the entries make_archive writes for the tree, in the order of os.walk with every directory
    listed sorted -- a symlink to a directory a directory entry, a symlink to a file the file's entry --, the number
    of names it writes no entry for)"""
    children = {}
    for p in nodes:
        if p:
            children.setdefault(posixpath.dirname(p), []).append(p)
    out, skipped, stack = [], 0, [""]
    while stack:
        d = stack.pop()
        dirs, files = [], []
        for p in sorted(children.get(d, []), key=posixpath.basename):
            t = lookup(nodes, p)
            (dirs if isinstance(t, _Dir) else files).append((p, t))
        out += dirs
        for p, t in files:
            if isinstance(t, _File):
                out.append((p, t))
            else:
                skipped += 1
        stack += [p for p, _ in reversed(dirs) if isinstance(nodes[p], _Dir)]
    return out, skipped


def select(nodes):
    """(the files `find -name "*.so" | xargs strip` strips in the tree, each once, the *.so names it leaves alone)"""
    chosen, skipped = {}, 0
    for p in sorted(nodes):
        if p and posixpath.basename(p).endswith(Z.SO_SUFFIX):
            t = lookup(nodes, p)
            if isinstance(t, _File):
                chosen.setdefault(id(t), t)
            else:
                skipped += 1
    return sorted(chosen.values(), key=lambda f: f.position()), skipped


def zip_info(path, node, size, umask):
    """the ZipInfo ZipInfo.from_file (strict_timestamps=False) reads for the extracted file or directory"""
    isdir = isinstance(node, _Dir)
    mode = node.mode if node.mode is not None else 0o777 & ~umask
    mode = (stat.S_IFDIR if isdir else stat.S_IFREG) | (mode & 0o7777)
    date_time = time.localtime(node.mtime)[:6] if node.mtime is not None else (1980, 1, 1, 0, 0, 0)
    if date_time[0] < 1980:
        date_time = (1980, 1, 1, 0, 0, 0)
    elif date_time[0] > 2107:
        date_time = (2107, 12, 31, 23, 59, 59)
    zi = zipfile.ZipInfo(path + "/" if isdir else path, date_time)
    zi.external_attr = (mode & 0xFFFF) << 16 | (0x10 if isdir else 0)
    zi.file_size = 0 if isdir else size
    return zi


def zip_with(srcs, dst, reader, indexer, stripper, encoder, prefix="", fallback_host_strip=True,
             tolerate_non_elf=False, check=None, parser=None, resolver=None):
    """zip_tarballs with the engines given (tarball.GpuTarReader, tarball.GpuTarIndex, zipfile_gpu.GpuStripper,
    zipfile_gpu.GpuZipEncoder fed by submit_device and, with check, deps.GpuElfParser and deps.GpuSymbolResolver, or
    stand-ins with the same interfaces)."""
    srcs = [os.fspath(srcs)] if isinstance(srcs, (str, bytes, os.PathLike)) else [os.fspath(s) for s in srcs]
    dst = os.fspath(dst)
    check_prefix(prefix)
    check = _check_engines(check, parser, resolver)
    if not srcs:
        raise ValueError("zip_tarballs: no source")
    for s in srcs:
        if os.path.realpath(s) == os.path.realpath(dst) or (os.path.exists(dst) and os.path.samefile(s, dst)):
            raise ValueError("zip_tarballs: %r is a source being read; write the result somewhere else" % dst)
    if encoder.piece_bytes < Z.CHUNK:
        raise ValueError("pieces of %d bytes: at least %d are needed" % (encoder.piece_bytes, Z.CHUNK))
    refs = reader.read_many(srcs)
    listings, index = [], {"kernel_ms": 0.0, "n_members": 0, "ranges": 0, "bytes": 0, "misses": 0, "miss_bytes": 0}
    views = []
    for ref in refs:
        members, _, view, (ranges, data, ist) = T.list_members(ref, indexer, reader)
        listings.append(members)
        views.append(view)
        index["kernel_ms"] += ist.get("kernel_ms", 0.0)
        index["n_members"] += ist.get("n_members", len(members))
        index["ranges"] += len(ranges)
        index["bytes"] += len(data)
    nodes = merge(listings, prefix)
    entries, skipped_entries = walk(nodes)
    chosen, skipped = select(nodes)

    def source(f):
        return refs[f.src][0] + f.member.offset_data, f.member.size
    res = stripper.strip([source(f) for f in chosen]) if chosen else []
    data_of, c = {}, {"gpu": 0, "fallback": 0, "skipped": skipped, "in_bytes": 0, "out_bytes": 0}
    for f, (status, ref) in zip(chosen, res):
        if status == N.ST_OK:
            c["gpu"] += 1
        elif status == N.ST_NOT_ELF and tolerate_non_elf:
            c["skipped"] += 1
            continue
        else:
            old = stripper.fetch(source(f))
            fixed = stripper.host_strip(old) if fallback_host_strip else None
            if fixed is None:
                if tolerate_non_elf and old[:4] != b"\x7fELF":
                    c["skipped"] += 1
                    continue
                raise Z.StripFailed(f.member.name, "strip refuses this file (the reference's xargs exits 123)"
                                    if fallback_host_strip else "not stripped on the GPU, and the host strip is off")
            c["fallback"] += 1
            ref = stripper.upload(fixed)
        data_of[id(f)] = ref
        c["in_bytes"] += f.member.size
        c["out_bytes"] += ref[1]

    umask = Z._umask()
    items, infos = [], []
    for i, (p, node) in enumerate(entries):
        ref = data_of.get(id(node)) or source(node) if isinstance(node, _File) else None
        infos.append((None, zip_info(p, node, ref[1] if ref else 0, umask)))
        if ref is not None:
            items.append((i, ref))
    report = None
    if check is not None:
        report = check_layer(check, [zi for _, zi in infos], dict(items), {}, None, parser, resolver)

    out_dir = os.path.dirname(dst) or "."
    os.makedirs(out_dir, exist_ok=True)
    fd, tmp = tempfile.mkstemp(prefix=os.path.basename(dst) + ".", suffix=".tmp", dir=out_dir)
    downloaded = 0
    try:
        with os.fdopen(fd, "w+b") as fp:
            w = Z._ContainerWriter(fp, infos)
            in_flight = []

            def collect():
                nonlocal downloaded
                body, res = encoder.collect()
                downloaded += len(body)
                chunks = getattr(encoder, "seek_chunks", None) or [None] * len(res)
                for (idx, (_, nbytes)), (off, k, crc, ended), ch in zip(in_flight.pop(0), res, chunks):
                    w.part(idx, body[off:off + k], crc, ended, nbytes, ch)

            for segs, flags in Z._device_pieces(items, encoder.piece_bytes, encoder.max_segs):
                encoder.submit_device([ref for _, ref in segs], flags)
                in_flight.append(segs)
                if len(in_flight) == 2:
                    collect()
            while in_flight:
                collect()
            w.finish()
            zip_bytes = fp.tell()
        os.chmod(tmp, 0o666 & ~umask)
        os.replace(tmp, dst)
    except BaseException:
        os.unlink(tmp)
        raise
    index["misses"] = sum(v.misses for v in views)
    index["miss_bytes"] = sum(v.miss_bytes for v in views)
    st = {"sources": len(srcs), "members": sum(len(m) for m in listings), "entries": len(infos),
          "files": w.n_files, "skipped_entries": skipped_entries, "selected": len(chosen), "gpu": c["gpu"],
          "fallback": c["fallback"], "skipped": c["skipped"], "in_bytes": c["in_bytes"], "out_bytes": c["out_bytes"],
          "file_bytes": w.in_bytes, "deflated_bytes": w.out_bytes, "tar_bytes_in": sum(n for _, n in refs),
          "src_bytes": sum(os.path.getsize(s) for s in srcs), "zip_bytes": zip_bytes,
          "uploaded_bytes": reader.uploaded + stripper.uploaded,
          "downloaded_bytes": reader.downloaded + 16 * index["ranges"] + index["bytes"] + downloaded +
          stripper.downloaded,
          "index": index, "inflate": reader.stats(), "strip": stripper.stats(), "deflate": encoder.stats()}
    st["kernel_ms"] = (st["inflate"].get("kernel_ms", 0.0) + index["kernel_ms"] + sum(st["strip"].values()) +
                       st["deflate"].get("kernel_ms", 0.0))
    if report is not None:
        st["check"] = report
    return st


def _check_engines(check, parser, resolver):
    """check validated before any source is read (deps.check_options), and the engines it needs present"""
    if check is None:
        return None
    check = D.check_options(check)
    if parser is None or ((check.get("symbols") or check.get("python")) and resolver is None):
        raise ValueError("check needs a parser, and a resolver with symbols=True or python")
    return check


def check_layer(check, infos, resident, wheel_members, decoder, parser, resolver):
    """deps.check_entries(**check) over a zip before any of it is written: infos [ZipInfo] are its entries, resident
    {entry index: (device address, size)} the entries whose bytes the writer holds on the device (the stripped
    objects, the tar arena, the host upload) and wheel_members {entry index: (ZipInfo, (ZipFile, open file, size))}
    the entries whose DEFLATE body is copied from a wheel, inflated by decoder when a closure reaches them.  Returns the
    report check_zip gives for the zip, its stats with inflate_ms (those inflates only) and roots_reused (the roots
    whose bytes were already on the device); raises deps.CheckFailed when it has problems."""
    entries = [(i, zi.filename, None) for i, zi in enumerate(infos)]   # a symlink is written as a file entry
    later = D.member_decoder(decoder, parser, wheel_members)
    ms0 = decoder.stats().get("kernel_ms", 0.0) if decoder is not None else 0.0

    def decode(keys, consume):
        here = [k for k in keys if k in resident]
        if here:
            consume(here, [resident[k] for k in here])
        rest = [k for k in keys if k not in resident]
        return later(rest, consume) if rest else 0
    report = D.check_entries(entries, decode, parser, resolver=resolver, **check)
    st = report["stats"]
    st["inflate_ms"] = decoder.stats().get("kernel_ms", 0.0) - ms0 if decoder is not None else 0.0
    st["roots_reused"] = sum(1 for i, zi in enumerate(infos) if i in resident and Z.selected_for_strip(zi))
    if report["problems"]:
        raise D.CheckFailed(report)
    return report


def zip_tarballs(srcs, dst, prefix="", ctx=None, compresslevel=None, fallback_host_strip=True, tolerate_non_elf=False,
                 piece_bytes=PIECE_BYTES, seek_table=False, check=None):
    """Write the Lambda zip `dst` of the package tarballs `srcs` (one .tar.gz path or a list), every shared object
    stripped, without unpacking them: entry for entry the zip that these passes give --
    `tarfile.open(src, "r:gz").extractall(tree / prefix, filter="fully_trusted")` for each source in order,
    `find tree -name "*.so" | xargs strip`, `shutil.make_archive` of tree -- with the entries in the order of os.walk
    listing every directory sorted, so the same sources always give the same bytes.  prefix: "" for a function
    bundle, "python/" for a layer; it must be empty or end in "/", without ".." or a leading "/".

    Entries: a directory (every prefix component included) is a ZIP_STORED directory entry; a regular file, a hard
    link and a symlink resolving to a file inside the tree are ZIP_DEFLATED entries with that file's bytes (stored once
    per name, as make_archive follows links); a symlink resolving to a directory is a directory entry that is not
    descended into; dangling symlinks, symlinks leaving the tree, FIFOs and devices get no entry (skipped_entries).
    external_attr and date_time are what ZipInfo.from_file reads from the extracted tree, with tarfile's order of
    effects (a hard link's mode and mtime apply to the file it shares; a directory member's after its source's
    files).  Deviations, where the passes would record the time they ran: timestamps outside 1980-2107 are clamped as
    ZipFile(strict_timestamps=False) clamps them (make_archive raises); a stripped file keeps its member's mtime, as
    `strip -p`; a directory with no member gets 1980-01-01 00:00:00 and mode 0o777 & ~umask; a directory a later
    source adds to keeps its last directory member's mtime.  The entries do not depend on who runs the call: a
    directory member without search permission (mode 0o644, say) still lists the files below it, which the passes run
    by an ordinary user would lose because make_archive cannot stat them.

    Several sources merge as consecutive extractalls: a later member replaces an earlier one of the same name, which
    is accepted for a directory onto a directory and a regular file onto a regular file only; any other collision,
    replacing a file that a hard link shares, a sparse member or a member below a symlink raises ValueError before dst
    is created.  The `*.so` names of the merged tree select the files to strip (through links, as GNU strip writes
    through them); each is stripped once however many entries show it.

    Bodies are what zip_tree writes for the same file bytes at the same compresslevel and piece_bytes;
    seek_table=True gives multi-chunk members a seek table in the central directory, as zip_tree does.  Sources with
    a seek table are read from it.  fallback_host_strip, tolerate_non_elf, StripFailed, framing and data errors and
    NativeError(LB2_E_CAPACITY) behave as in tarball.strip_tarball.  dst appears when it is complete and not at all
    when the call raises; a dst that is one of the sources raises ValueError.

    Returns a stats dict: sources, members, entries, files, skipped_entries; selected, gpu, fallback, skipped; in_bytes
    / out_bytes (the stripped files before and after), file_bytes (every file entry's bytes), deflated_bytes (their
    bodies), tar_bytes_in, src_bytes, zip_bytes; uploaded_bytes / downloaded_bytes (everything that crossed the bus);
    index, inflate, strip and deflate (the engines' stats) and kernel_ms, their kernel times summed.

    check (a dict of check_zip's keyword arguments: mount, arch, provided, max_versions, ld_library_path, symbols,
    interpreter, runtime_libs, python) checks the zip before it is written, on the stripped objects where they lie on the
    device (DESIGN.md section 9.10): stats["check"] is the report check_zip(dst, **check) would return, with stats
    roots_reused added, and a report with problems raises deps.CheckFailed (its report attached) before dst is
    created or replaced.  An unknown key or a refused value raises ValueError before any source is read.  There is
    no CPU path: without a GPU this raises."""
    N.deflate_flags(compresslevel)
    check_prefix(prefix)
    if check is not None:
        D.check_options(check)
    own = False
    if ctx is None:
        ctx, own = T._default_context()
    try:
        with T.GpuTarReader(ctx) as reader, Z.GpuStripper(ctx) as stripper, \
                Z.GpuZipEncoder(ctx, piece_bytes, compresslevel=compresslevel, host_buffers=False,
                                seek_table=seek_table) as enc, _check_engine_set(ctx, check) as (parser, resolver):
            return zip_with(srcs, dst, reader, T.GpuTarIndex(ctx), stripper, enc, prefix, fallback_host_strip,
                            tolerate_non_elf, check, parser, resolver)
    finally:
        if own:
            ctx.close()


@contextlib.contextmanager
def _check_engine_set(ctx, check):
    """(GpuElfParser, GpuSymbolResolver) for check, each None where check does not need it"""
    with contextlib.ExitStack() as stack:
        parser = stack.enter_context(D.GpuElfParser(ctx)) if check is not None else None
        resolver = stack.enter_context(D.GpuSymbolResolver(ctx)) \
            if check is not None and (check.get("symbols") or check.get("python")) else None
        yield parser, resolver


# ---- zip_build: prebuilt tarballs and wheels, pip's target install and the build script's clean-up ----------------
# pip is not run.  What `pip install --no-deps --no-index --target T W1.whl ...` (pip 24) does to the tree is restated
# on the merged tree's nodes: every wheel is installed into a temporary home H (the scheme get_scheme(name, home=H)
# gives), then the top-level items of H/lib/python and of H are moved into T as commands/install.py's
# _handle_target_dir moves them.  Only the parts of pip that decide names, bytes and modes are restated; the RECORD,
# INSTALLER, REQUESTED and direct_url.json files pip writes go with the .dist-info directory the clean-up removes.

_WHEEL_FILE = re.compile(r"^(?P<name>[^\s-]+?)-(?P<ver>[^\s-]*?)(-(?P<build>\d[^-]*?))?-(?P<pyver>[^\s-]+?)"
                         r"-(?P<abi>[^\s-]+?)-(?P<plat>[^\s-]+?)\.whl$")   # pip's Wheel.wheel_file_re
_ENTRY = re.compile(r"(?P<name>([^\[]\S*))\s*=\s*(?P<callable>(\w+)([:\.]\w+)*)"
                    r"\s*(\[\s*(?P<flags>[\w-]+(=\w+)?(,\s*\w+(=\w+)?)*)\s*\])?")   # distlib's ENTRY_RE
_LAUNCHER = r"""# -*- coding: utf-8 -*-
import re
import sys
from %(module)s import %(import_name)s
if __name__ == '__main__':
    sys.argv[0] = re.sub(r'(-script\.pyw|\.exe)?$', '', sys.argv[0])
    sys.exit(%(func)s())
"""                                                                   # distlib's SCRIPT_TEMPLATE, as pip 24 writes it
_LIB = "lib/python"                                                   # purelib and platlib under the home
BUILD_DIR = "./build/"   # the directory the reference's clean-up lines print paths under (`find ./build/ -name tests`)


class _WheelFile(_File):
    """a file pip installs: a wheel member (data None: its body is copied or decoded) or bytes made on the host (a
    `#!python` script fixed, a console or gui script generated); date_time is the entry's"""

    def __init__(self, src, member, mode, date_time, data=None):
        super().__init__()
        self.src, self.member, self.mode, self.date_time, self.data = src, member, mode, date_time, data

    def position(self):
        return self.src, self.member.header_offset if self.data is None else 1 << 62

    def label(self):
        return self.member.filename if self.member is not None else "a generated script"

    def signature(self):
        if self.data is not None:
            return len(self.data), zlib.crc32(self.data), self.mode
        return self.member.file_size, self.member.CRC, self.mode


def canonical_name(name):
    return re.sub(r"[-_.]+", "-", name).lower()


def _shebang(executable):
    """distlib's shebang for pip's console and gui scripts: the interpreter quoted when it holds a space, and the
    /bin/sh trampoline when the line would hold a space or pass 127 bytes"""
    if " " in executable and not executable.startswith('"'):
        if executable.startswith("/usr/bin/env "):
            env, rest = executable.split(" ", 1)
            if " " in rest and not rest.startswith('"'):
                executable = '%s "%s"' % (env, rest)
        else:
            executable = '"%s"' % executable
    exe = executable.encode("utf-8")
    if b" " not in exe and len(exe) + 3 <= 127:
        return b"#!" + exe + b"\n"
    return b"#!/bin/sh\n'''exec' " + exe + b' "$0" "$@"\n' + b"' '''\n"


class _WheelMetadata(importlib.metadata.Distribution):
    """the wheel's .dist-info read from the archive, for its entry points as pip's importlib backend reads them"""

    def __init__(self, zf, info_dir):
        self._zf, self._info = zf, info_dir

    def read_text(self, filename):
        try:
            return self._zf.read(self._info + "/" + filename).decode("utf-8")
        except KeyError:
            return None

    def locate_file(self, path):
        raise NotImplementedError


def read_wheel(path, src, umask, executable=sys.executable):
    """(canonical name, {path under the temporary home: _WheelFile}) of what pip 24 installs from one wheel, checked
    before anything is written: ValueError for a name that is not a wheel's, not exactly one .dist-info directory, a
    Wheel-Version other than 1.x, a member leaving its scheme directory or under an unknown scheme key, a member that is
    encrypted or compressed with anything but stored or deflated, an entry point without a callable, and the entry
    points pip treats specially (pip, easy_install)."""
    m = _WHEEL_FILE.match(os.path.basename(path))
    if not m:
        raise ValueError("%s: not a wheel file name (name-version-python-abi-platform.whl)" % path)
    name = m.group("name").replace("_", "-")
    with zipfile.ZipFile(path) as zf:
        names = list(dict.fromkeys(zf.namelist()))     # a repeated name installs its last entry, as getinfo reads it
        info_dirs = sorted({n.split("/", 1)[0] for n in names if n.split("/", 1)[0].endswith(".dist-info")})
        if len(info_dirs) != 1:
            raise ValueError("%s: %d .dist-info directories, one is needed" % (path, len(info_dirs)))
        info_dir = info_dirs[0]
        if not canonical_name(info_dir).startswith(canonical_name(name)):
            raise ValueError("%s: .dist-info directory %r does not start with %r" % (path, info_dir, name))
        try:
            version = email.parser.Parser().parsestr(zf.read(info_dir + "/WHEEL").decode("utf-8"))["Wheel-Version"]
            major = int(version.strip().split(".")[0])
        except (KeyError, AttributeError, ValueError, UnicodeDecodeError):
            raise ValueError("%s: no valid Wheel-Version in %s/WHEEL" % (path, info_dir)) from None
        if major != 1:
            raise ValueError("%s: Wheel-Version %s, only 1.x is supported" % (path, version.strip()))
        scheme = {"purelib": _LIB, "platlib": _LIB, "scripts": "bin", "data": "",
                  "headers": "include/site/python%d.%d/%s" % (sys.version_info[0], sys.version_info[1], name)}
        meta = _WheelMetadata(zf, info_dir)
        eps = meta.entry_points
        console = {e.name: e.value for e in eps if e.group == "console_scripts"}
        gui = {e.name: e.value for e in eps if e.group == "gui_scripts"}
        if "pip" in console or "easy_install" in console:
            raise ValueError("%s: the entry points pip installs itself under several names are not supported" % path)

        def wrapper(base):
            low = base.lower()
            for suffix in (".exe", "-script.py", ".pya"):
                if low.endswith(suffix):
                    base = base[:-len(suffix)]
                    break
            return base in console or base in gui

        files = {}
        for n in names:
            if n.endswith("/"):
                continue
            zi = zf.getinfo(n)
            if zi.compress_type not in (zipfile.ZIP_STORED, zipfile.ZIP_DEFLATED) or zi.flag_bits & 0x1:
                raise ValueError("%s: member %r is encrypted or compressed with method %d; only stored and deflated "
                                 "members are read" % (path, n, zi.compress_type))
            normed = posixpath.normpath(n)
            if n.split("/", 1)[0].endswith(".data"):
                parts = normed.split("/", 2)
                if len(parts) < 3 or parts[1] not in scheme:
                    raise ValueError("%s: member %r is not under <name>.data/<scheme key>/ (purelib, platlib, "
                                     "headers, scripts, data)" % (path, n))
                key, rel = parts[1], parts[2]
            else:
                key, rel = "purelib", normed
            if T._leaves(rel) or rel in (".", ""):
                raise ValueError("%s: member %r leaves the directory it is installed to" % (path, n))
            dest = posixpath.join(scheme[key], rel) if scheme[key] else rel
            mode = stat.S_IMODE(zi.external_attr >> 16)
            executable_bit = bool(zi.external_attr >> 16 and stat.S_ISREG(zi.external_attr >> 16) and mode & 0o111)
            mode = 0o777 & ~umask | 0o111 if executable_bit else 0o666 & ~umask
            data = None
            parts = n.split("/", 2)
            if len(parts) > 2 and parts[0].endswith(".data") and parts[1] == "scripts":
                if wrapper(posixpath.basename(dest)):
                    continue                                  # the generated script takes its place
                body = zf.read(zi)
                first, nl, rest = body.partition(b"\n")
                if first.startswith(b"#!python"):             # pip's fix_script
                    data = b"#!" + os.fsencode(executable) + os.linesep.encode("ascii") + rest
            files[dest] = _WheelFile(src, zi, mode, zi.date_time, data)
        specs = [("%s = %s" % kv, False) for kv in console.items()] + [("%s = %s" % kv, True) for kv in gui.items()]
        when = zf.getinfo(info_dir + "/entry_points.txt").date_time if specs else None
        for spec, _ in specs:
            e = _ENTRY.search(spec)
            if not e or e.group("callable").count(":") != 1:
                raise ValueError("%s: entry point %r has no callable (module:function)" % (path, spec))
            module, func = e.group("callable").split(":")
            text = _shebang(executable) + (_LAUNCHER % {"module": module, "import_name": func.split(".")[0],
                                                         "func": func}).encode("utf-8")
            dest = "bin/" + e.group("name")
            if dest in files:
                raise ValueError("%s: entry point %r would overwrite a file of the wheel" % (path, e.group("name")))
            files[dest] = _WheelFile(src, None, 0o666 & ~umask | 0o555, when, text)
    return canonical_name(name), files


def read_home(wheels, umask=0o022, executable=sys.executable, first_src=0):
    """The temporary home `pip install --no-deps --no-index --target` installs the wheels into, before anything moves:
    ({path under the home: _WheelFile}, the number of scripts generated).  Two wheels may install the same path only
    with the same size, CRC-32 and mode (the first wheel's entry is kept); any other overlap, one distribution given
    twice and a path installed both as a file and as a directory raise ValueError, as read_wheel's refusals do."""
    home, seen, generated = {}, {}, 0
    for i, path in enumerate(wheels):
        name, files = read_wheel(path, first_src + i, umask, executable)
        if name in seen:
            raise ValueError("%s and %s install the same distribution %r" % (wheels[seen[name]], path, name))
        seen[name] = i
        generated += sum(1 for f in files.values() if f.member is None)
        for dest, f in files.items():
            old = home.get(dest)
            if old is not None and old.signature() != f.signature():
                raise ValueError("%s and %s both install %r with different contents or modes"
                                 % (wheels[old.src - first_src], path, dest))
            home.setdefault(dest, f)
    dirs = {posixpath.dirname(d) for d in home}
    for d in list(dirs):
        while d:
            d = posixpath.dirname(d)
            dirs.add(d)
    for d in dirs:
        if d in home:
            raise ValueError("%s: installed both as a file and as a directory" % d)
    return home, generated


def install(nodes, home, prefix=""):
    """Move the temporary home's items into the merged tree as pip's _handle_target_dir does without --upgrade: the
    top-level items of lib/python, then the home's other top-level items (lib excepted), an item whose name the target
    tree/prefix already holds skipped whole.  Returns the skipped item names."""
    dirs = set()
    for p in home:
        while p:
            p = posixpath.dirname(p)
            dirs.add(p)
    base = prefix[:-1]
    children = {}
    for p in list(home) + [d for d in dirs if d]:
        children.setdefault(posixpath.dirname(p), []).append(p)
    skipped = []
    for src_dir, skip in ((_LIB, lambda item: False), ("", lambda item: _LIB.startswith(item))):
        for item in sorted(posixpath.basename(p) for p in children.get(src_dir, [])):
            if skip(item):
                continue
            target = base + "/" + item if base else item
            if target in nodes:
                if lookup(nodes, target) is None:
                    raise ValueError("%r: the tree holds it as a dangling or looping symlink, which pip would replace"
                                     % target)
                skipped.append(item)
                continue
            origin = posixpath.join(src_dir, item) if src_dir else item
            todo = [origin]
            while todo:
                p = todo.pop()
                nodes[target + p[len(origin):]] = home.get(p) or _Dir()
                todo += children.get(p, [])
    return skipped


def clean(nodes, prefix="", keep_tests=()):
    """The build script's clean-up lines on tree/prefix, in the model: `*.egg-info` and `*.dist-info` at its top level
    (shell globs: no dot files), `__pycache__` at any depth, and `tests` at any depth unless the keep pattern
    (project_build._keep_pattern) matches the path `find ./build/ -name tests` prints, decided by the same regcomp rule
    as lb2_tree_cleanup.  Removes every node below a match; returns the matches per rule (a match below another
    counted once, with the outer one)."""
    from .project_build import _keep_pattern
    base = prefix[:-1]
    rel = {p: (p[len(base) + 1:] if base else p) for p in nodes if p and (not base or p.startswith(base + "/"))}
    hits, tests = {}, []
    for p, r in rel.items():
        leaf = posixpath.basename(r)
        if "/" not in r and not r.startswith(".") and r.endswith((".egg-info", ".dist-info")):
            hits[p] = r.rsplit(".", 1)[1]
        elif leaf == "__pycache__":
            hits[p] = "__pycache__"
        elif leaf == "tests":
            tests.append(p)
    if tests:
        lib = N.load()
        lines = (C.c_char_p * len(tests))(*[os.fsencode(BUILD_DIR + rel[p]) for p in tests])
        out = (C.c_uint8 * len(tests))()
        rc = lib.lb2_cleanup_tests_removed(os.fsencode(_keep_pattern(keep_tests)), lines, len(tests), out)
        if rc != N.LB2_OK:
            raise ValueError("keep_tests %r: not a valid grep pattern" % (list(keep_tests),))
        hits.update((p, "tests") for p, r in zip(tests, out) if r)
    counts = {"egg-info": 0, "dist-info": 0, "__pycache__": 0, "tests": 0, "entries": 0}

    def under(p):
        while p != base and p:
            p = posixpath.dirname(p)
            if p in hits:
                return True
        return False
    for p in [p for p in rel if p in hits or under(p)]:
        if p in hits and not under(p):
            counts[hits[p]] += 1
        counts["entries"] += 1
        del nodes[p]
    return counts


def _entry_info(path, node, size, umask):
    if not isinstance(node, _WheelFile):
        return zip_info(path, node, size, umask)
    zi = zipfile.ZipInfo(path, node.date_time)
    zi.external_attr = (stat.S_IFREG | node.mode) << 16
    zi.file_size = size
    return zi


def build_with(dst, tarballs, wheels, reader, indexer, decoder, stripper, encoder, prefix="", keep_tests=(),
               executable=sys.executable, fallback_host_strip=True, tolerate_non_elf=False, check=None, parser=None,
               resolver=None):
    """zip_build with the engines given (tarball.GpuTarReader, tarball.GpuTarIndex, zipfile_gpu.GpuUnzipDecoder,
    zipfile_gpu.GpuStripper, zipfile_gpu.GpuZipEncoder fed by submit_device and, with check, deps.GpuElfParser and
    deps.GpuSymbolResolver, or stand-ins with the same interfaces)."""
    tarballs, wheels = [os.fspath(t) for t in tarballs], [os.fspath(w) for w in wheels]
    dst = os.fspath(dst)
    check_prefix(prefix)
    check = _check_engines(check, parser, resolver)
    if not tarballs and not wheels:
        raise ValueError("zip_build: no tarball and no wheel")
    for s in tarballs + wheels:
        if os.path.realpath(s) == os.path.realpath(dst) or (os.path.exists(dst) and os.path.samefile(s, dst)):
            raise ValueError("zip_build: %r is a source being read; write the result somewhere else" % dst)
    if encoder.piece_bytes < Z.CHUNK:
        raise ValueError("pieces of %d bytes: at least %d are needed" % (encoder.piece_bytes, Z.CHUNK))
    umask = Z._umask()
    home, generated = read_home(wheels, umask, executable, len(tarballs))      # a wheel's refusal comes first
    refs = reader.read_many(tarballs) if tarballs else []
    listings, views = [], []
    index = {"kernel_ms": 0.0, "n_members": 0, "ranges": 0, "bytes": 0, "misses": 0, "miss_bytes": 0}
    for ref in refs:
        members, _, view, (ranges, data, ist) = T.list_members(ref, indexer, reader)
        listings.append(members)
        views.append(view)
        index["kernel_ms"] += ist.get("kernel_ms", 0.0)
        index["n_members"] += ist.get("n_members", len(members))
        index["ranges"] += len(ranges)
        index["bytes"] += len(data)
    nodes = merge(listings, prefix)
    skipped_items = install(nodes, home, prefix)
    removed = clean(nodes, prefix, keep_tests)
    entries, skipped_entries = walk(nodes)
    chosen, skipped = select(nodes)
    chosen_ids = {id(f) for f in chosen}

    c = {"gpu": 0, "fallback": 0, "skipped": skipped, "in_bytes": 0, "out_bytes": 0, "uploaded": 0}
    dev, host = {}, {}          # id(node) -> its bytes for the zip: a device ref / bytes to upload after the strip
    # the decoder's output lives until its next run; the check's later rounds run it again, so with a check a member
    # left unstripped in that output (a stored member, a non-ELF `*.so` under tolerate_non_elf) goes up with the host's
    keep_decoded = check is None

    def host_fix(data, name):
        fixed = stripper.host_strip(data) if fallback_host_strip else None
        if fixed is None:
            if tolerate_non_elf and data[:4] != b"\x7fELF":
                c["skipped"] += 1
                return data
            raise Z.StripFailed(name, "strip refuses this file (the reference's xargs exits 123)"
                                if fallback_host_strip else "not stripped on the GPU, and the host strip is off")
        c["fallback"] += 1
        c["in_bytes"] += len(data)
        c["out_bytes"] += len(fixed)
        return fixed

    def strip(pairs, keep_on_device):
        """strip [(node, device ref)] in one batch; the results go to dev, or to host when the refs die next"""
        res = stripper.strip([r for _, r in pairs]) if pairs else []
        for (f, r), (status, new) in zip(pairs, res):
            if status == N.ST_OK:
                c["gpu"] += 1
                c["in_bytes"] += r[1]
                c["out_bytes"] += new[1]
                if keep_on_device:
                    dev[id(f)] = new
                else:
                    host[id(f)] = stripper.fetch(new)
            elif status == N.ST_NOT_ELF and tolerate_non_elf:
                c["skipped"] += 1
                if keep_on_device and (keep_decoded or not isinstance(f, _WheelFile)):
                    dev[id(f)] = r
                else:
                    host[id(f)] = stripper.fetch(r)
            else:
                host[id(f)] = host_fix(stripper.fetch(r), f.label())

    # the wheel members decoded on the device: the selected ones, and stored ones (their bodies are no DEFLATE)
    files = {id(t): t for _, t in entries if isinstance(t, _File)}
    files.update((id(f), f) for f in chosen)
    todo = sorted((f for f in files.values() if isinstance(f, _WheelFile) and f.data is None and
                   (id(f) in chosen_ids or f.member.compress_type != zipfile.ZIP_DEFLATED)),
                  key=lambda f: f.position())
    handles = [open(w, "rb") for w in wheels]
    zfs = [zipfile.ZipFile(h) for h in handles]
    try:
        sources = []
        for zf, h in zip(zfs, handles):
            h.seek(0, os.SEEK_END)
            sources.append((zf, h, h.tell()))
        tar_chosen = [(f, (refs[f.src][0] + f.member.offset_data, f.member.size)) for f in chosen
                      if not isinstance(f, _WheelFile)]
        by_id, tar_done = {id(f): f for f in todo}, []

        def decoded(part, got, whole):
            for key, zi, _ in part:
                status = got.get(key, (Z.UNZIP_OK, None))[0]
                if status != Z.UNZIP_OK:
                    raise Z.BadZipMember(zi.filename, {Z.UNZIP_BAD_DATA: "Invalid DEFLATE data", Z.UNZIP_BAD_CRC:
                                                       "Bad CRC-32", Z.UNZIP_WRONG_SIZE: "Wrong uncompressed size"}[status])
            pairs = []
            for key, zi, (zf, _, _) in part:
                f = by_id[key]
                if key not in got:                            # not on the device: read by the stdlib
                    data = zf.read(zi)
                    host[key] = host_fix(data, zi.filename) if key in chosen_ids else data
                elif key in chosen_ids:
                    pairs.append((f, got[key][1]))
                elif whole and keep_decoded:
                    dev[key] = got[key][1]
                else:
                    host[key] = stripper.fetch(got[key][1])
            if whole:                                         # every selected file in one strip batch
                strip(tar_chosen + pairs, True)
                tar_done.append(True)
            else:
                strip(pairs, False)
        batch = [(id(f), f.member, sources[f.src - len(tarballs)]) for f in todo]
        if batch:
            c["uploaded"] += Z.decode_members(decoder, batch, decoded)
        if not tar_done:                                      # no wheel member, or the wheels' batch was split
            strip(tar_chosen, True)
        for f in chosen:                                      # a script made on the host, named *.so
            if isinstance(f, _WheelFile) and f.data is not None:
                host[id(f)] = host_fix(f.data, f.label())
        for f in files.values():
            if isinstance(f, _WheelFile) and f.data is not None and id(f) not in host:
                host[id(f)] = f.data
        if host:                                              # one upload for every file made on the host
            buf, at = bytearray(), {}
            for k, data in host.items():
                buf += bytes(-len(buf) % Z.ALIGN)
                at[k] = (len(buf), len(data))
                buf += data
            addr = reader.upload(bytes(buf))
            for k, (off, n) in at.items():
                dev[k] = (addr + off, n)

        items, infos, copied = [], [], {}
        for i, (p, node) in enumerate(entries):
            ref = None
            if isinstance(node, _File):
                ref = dev.get(id(node))
                if ref is None and not isinstance(node, _WheelFile):
                    ref = (refs[node.src][0] + node.member.offset_data, node.member.size)
            if ref is not None:
                items.append((i, ref))
                infos.append((None, _entry_info(p, node, ref[1], umask)))
            elif isinstance(node, _WheelFile):                # a DEFLATE body copied from its wheel
                zi = _entry_info(p, node, node.member.file_size, umask)
                zi.compress_type, zi.CRC, zi.compress_size = zipfile.ZIP_DEFLATED, node.member.CRC, node.member.compress_size
                copied[i] = node
                infos.append((None, zi))
            else:
                infos.append((None, _entry_info(p, node, 0, umask)))
        report, unzip = None, decoder.stats()          # the build's decodes; the check's are in its report
        if check is not None:
            report = check_layer(check, [zi for _, zi in infos], dict(items),
                                 {i: (node.member, sources[node.src - len(tarballs)]) for i, node in copied.items()},
                                 decoder, parser, resolver)

        out_dir = os.path.dirname(dst) or "."
        os.makedirs(out_dir, exist_ok=True)
        fd, tmp = tempfile.mkstemp(prefix=os.path.basename(dst) + ".", suffix=".tmp", dir=out_dir)
        downloaded = 0
        try:
            with os.fdopen(fd, "w+b") as fp:
                position = {id(zi): i for i, (_, zi) in enumerate(infos)}

                def copy(zi):
                    node = copied.get(position[id(zi)])
                    if node is None:                          # a directory
                        zi.compress_size = zi.CRC = 0
                        fp.write(zi.FileHeader(False))
                        return
                    zf, h, _ = sources[node.src - len(tarballs)]
                    start = _body_offset(h, node.member)
                    fp.write(zi.FileHeader())
                    h.seek(start)
                    left = node.member.compress_size
                    while left:
                        block = h.read(min(left, 1 << 20))
                        if not block:
                            raise zipfile.BadZipFile("%s ends inside the body of %r" % (zf.filename, node.member.filename))
                        fp.write(block)
                        left -= len(block)

                w = Z._ContainerWriter(fp, infos, copy=copy)
                for i, node in copied.items():                # a body copied as it is keeps its seek table
                    field = ST.zip_field_of(node.member.extra)
                    if field:
                        w.tables[i] = field
                in_flight = []

                def collect():
                    nonlocal downloaded
                    body, res = encoder.collect()
                    downloaded += len(body)
                    chunks = getattr(encoder, "seek_chunks", None) or [None] * len(res)
                    for (idx, (_, nbytes)), (off, k, crc, ended), ch in zip(in_flight.pop(0), res, chunks):
                        w.part(idx, body[off:off + k], crc, ended, nbytes, ch)

                for segs, flags in Z._device_pieces(items, encoder.piece_bytes, encoder.max_segs):
                    encoder.submit_device([ref for _, ref in segs], flags)
                    in_flight.append(segs)
                    if len(in_flight) == 2:
                        collect()
                while in_flight:
                    collect()
                w.finish()
                zip_bytes = fp.tell()
            os.chmod(tmp, 0o666 & ~umask)
            os.replace(tmp, dst)
        except BaseException:
            os.unlink(tmp)
            raise
    finally:
        for zf in zfs:
            zf.close()
        for h in handles:
            h.close()
    index["misses"] = sum(v.misses for v in views)
    index["miss_bytes"] = sum(v.miss_bytes for v in views)
    n_copied = len(copied)
    st = {"sources": len(tarballs), "wheels": len(wheels), "members": sum(len(m) for m in listings),
          "wheel_members": sum(1 for z in zfs for zi in z.infolist() if not zi.is_dir()),
          "entries": len(infos), "files": w.n_files + n_copied, "skipped_entries": skipped_entries,
          "selected": len(chosen), "gpu": c["gpu"], "fallback": c["fallback"], "skipped": c["skipped"],
          "in_bytes": c["in_bytes"], "out_bytes": c["out_bytes"],
          "copied": {"members": n_copied, "bytes": sum(n.member.compress_size for n in copied.values()),
                     "file_bytes": sum(n.member.file_size for n in copied.values())},
          "generated_scripts": generated, "removed": removed, "skipped_items": skipped_items,
          "file_bytes": w.in_bytes, "deflated_bytes": w.out_bytes, "tar_bytes_in": sum(n for _, n in refs),
          "src_bytes": sum(os.path.getsize(s) for s in tarballs + wheels), "zip_bytes": zip_bytes,
          "uploaded_bytes": reader.uploaded + c["uploaded"] + stripper.uploaded,
          "downloaded_bytes": reader.downloaded + 16 * index["ranges"] + index["bytes"] + downloaded +
          stripper.downloaded,
          "index": index, "inflate": reader.stats() if tarballs else {}, "unzip": unzip,
          "strip": stripper.stats(), "deflate": encoder.stats()}
    st["kernel_ms"] = (st["inflate"].get("kernel_ms", 0.0) + index["kernel_ms"] + st["unzip"].get("kernel_ms", 0.0) +
                       sum(st["strip"].values()) + st["deflate"].get("kernel_ms", 0.0))
    if report is not None:
        st["check"] = report
    return st


def _body_offset(f, zi):
    """the offset of zi's body in the open archive f, from its local header"""
    f.seek(zi.header_offset)
    fh = f.read(zipfile.sizeFileHeader)
    if len(fh) != zipfile.sizeFileHeader or fh[:4] != zipfile.stringFileHeader:
        raise zipfile.BadZipFile("Bad magic number for file header of %r" % zi.filename)
    fh = struct.unpack(zipfile.structFileHeader, fh)
    return zi.header_offset + zipfile.sizeFileHeader + fh[zipfile._FH_FILENAME_LENGTH] + fh[zipfile._FH_EXTRA_FIELD_LENGTH]


def zip_build(dst, tarballs=(), wheels=(), prefix="", keep_tests=(), executable=sys.executable, ctx=None,
              compresslevel=None, fallback_host_strip=True, tolerate_non_elf=False, piece_bytes=PIECE_BYTES,
              seek_table=False, check=None):
    """Write the Lambda zip `dst` of a whole build -- prebuilt package tarballs and wheels -- as `lambdipy build`
    leaves it, without unpacking anything: entry for entry the zip these passes give, with T = tree / prefix:
    `tarfile.open(t, "r:gz").extractall(T, filter="fully_trusted")` for each tarball in order, `pip install --no-deps
    --no-index --target T W1.whl W2.whl ...` (pip 24, no --upgrade), the build script's clean-up lines on T (`rm -rf
    *.egg-info *.dist-info`, `find -name __pycache__ | xargs rm -rf`, `find -name tests | grep -v PATTERN | xargs rm
    -rf` with PATTERN project_build._keep_pattern(keep_tests)), `find T -name "*.so" | xargs strip`, and
    `shutil.make_archive` of tree, the entries in the order of os.walk listing every directory sorted.

    pip is restated on a model of the tree, not run (read_wheel, read_home, install): root members and
    <name>.data/{purelib,platlib} go to lib/python of a temporary home, scripts to bin, headers to
    include/site/pythonX.Y/<name>, data to the home itself; a `.data/scripts` file starting `#!python` gets
    `#!<executable>` (pip's fix_script); console and gui entry points become scripts in bin with pip 24's launcher
    text.  A member with an executable bit gets mode 0o777 & ~umask | 0o111, any other file 0o666 & ~umask (a fixed
    script keeps its member's rule), a generated script 0o666 & ~umask | 0o555 (distlib's set_mode).  The home's
    lib/python items, then its other top-level items (lib excepted), move into T; an item T already holds (from a
    tarball) is skipped whole, as pip warns and skips without --upgrade (stats skipped_items).  Two wheels may install
    the same path only with the same size, CRC-32 and mode (the entry keeps the first wheel's date); any other
    overlap, a distribution given twice, a wheel without exactly one .dist-info or with a Wheel-Version other than
    1.x, a member leaving the tree, an encrypted member or one compressed with anything but stored or deflated, and
    the tarball merges zip_tarballs refuses raise ValueError before dst exists.  Compatibility tags are not checked:
    the wheels are the ones downloaded for Lambda's platform.  The clean-up covers the tarballs' files too.

    Data path: a wheel file that is not stripped keeps its DEFLATE body, copied from the wheel with the CRC-32 and
    sizes of its central directory (its CRC is not checked, as in zipfile_gpu.strip_zip); it never crosses the bus.
    The `*.so` files select chooses in the final tree are stripped on the GPU: the wheel members among them (and any
    stored member) are uploaded in one buffer and inflated in one decoder run (zipfile_gpu.decode_members, split in
    halves when the device is too small), then stripped in one batch with the tarballs' files, with the host-strip
    fallback.  Scripts made on the host are uploaded once.  Every rewritten body is deflated on the GPU; compresslevel
    and seek_table apply to those bodies.

    Deviations, where the passes would record the time they ran: zip_tarballs' list, and a wheel file keeps its
    member's date_time, a generated script takes the date_time of its wheel's entry_points.txt, a directory pip makes
    gets 1980-01-01 00:00:00 and 0o777 & ~umask, and a directory that loses children to the clean-up keeps its own
    date.  Entry points named pip or easy_install (which pip installs under several names) raise ValueError.

    Returns zip_tarballs' stats dict with wheels, wheel_members, copied (members, bytes, file_bytes),
    generated_scripts, removed (the clean-up's matches per rule and the entries removed), skipped_items and unzip (the
    decoder's stats for the build) added.

    check is zip_tarballs' (DESIGN.md section 9.10): the roots are checked where the strip left them, the tarballs'
    files in the tar arena, and a wheel member that only a closure reaches (a `.libs/*.so.N`, whose body is otherwise
    copied) is inflated by the same decoder for the check alone.  With a check, a wheel member left unstripped in the
    decoder's output goes up with the files made on the host instead, since the check's inflates reuse that output.
    There is no CPU path: without a GPU this raises."""
    N.deflate_flags(compresslevel)
    check_prefix(prefix)
    if check is not None:
        D.check_options(check)
    own = False
    if ctx is None:
        ctx, own = T._default_context()
    try:
        with T.GpuTarReader(ctx) as reader, Z.GpuUnzipDecoder(ctx) as dec, Z.GpuStripper(ctx) as stripper, \
                Z.GpuZipEncoder(ctx, piece_bytes, compresslevel=compresslevel, host_buffers=False,
                                seek_table=seek_table) as enc, _check_engine_set(ctx, check) as (parser, resolver):
            return build_with(dst, tarballs, wheels, reader, T.GpuTarIndex(ctx), dec, stripper, enc, prefix,
                              keep_tests, executable, fallback_host_strip, tolerate_non_elf, check, parser, resolver)
    finally:
        if own:
            ctx.close()


def main(argv=None):
    """python -m lambdipy_b200.layer DST [SRC ...] [--wheel WHL ...] [--keep-tests NAME ...] [--clean]
    [--prefix python/] [--level 9] [--seek-table] [--check [the options of python -m lambdipy_b200.deps]]

    With --check, exit status 1 when the check finds problems (no zip is written) and 2 on a refused input."""
    import argparse
    ap = argparse.ArgumentParser(prog="python -m lambdipy_b200.layer",
                                 description="write the Lambda zip of .tar.gz package assets, shared objects stripped, "
                                             "inflated, stripped and deflated on the GPU")
    ap.add_argument("dst")
    ap.add_argument("srcs", nargs="*", metavar="src")
    ap.add_argument("--wheel", action="append", default=[], metavar="WHL",
                    help="install this wheel as `pip install --no-deps --target` would (repeatable; implies --clean)")
    ap.add_argument("--keep-tests", action="append", default=[], metavar="NAME",
                    help="keep the tests directories whose path contains NAME (repeatable)")
    ap.add_argument("--clean", action="store_true",
                    help="run the build script's clean-up lines (*.egg-info, *.dist-info, __pycache__, tests)")
    ap.add_argument("--prefix", default="", help='directory of the zip the sources go under ("python/" for a layer)')
    ap.add_argument("--level", type=int, choices=[9], default=None, help="9: the optimal parse (smaller, slower)")
    ap.add_argument("--seek-table", action="store_true",
                    help="give multi-chunk members seek tables, with which the GPU reader decodes them without search")
    ap.add_argument("--check", action="store_true",
                    help="check that the shared objects will load on Lambda, as python -m lambdipy_b200.deps does, "
                         "before the zip is written; on a problem no zip is written (the options below need it)")
    check_dests = D.add_check_arguments(ap)
    args = ap.parse_args(argv)
    if not args.srcs and not args.wheel:
        ap.error("give at least one tarball or --wheel")
    if not args.check and any(getattr(args, k) != ap.get_default(k) for k in check_dests):
        ap.error("--mount, --arch, --provided, --max-version, --ld-library-path, --symbols, --interpreter, "
                 "--runtime-lib and --python need --check")
    try:
        kw = {"check": D.check_kwargs(args)} if args.check else {}
        if args.wheel or args.clean:
            st = zip_build(args.dst, args.srcs, args.wheel, prefix=args.prefix, keep_tests=args.keep_tests,
                           compresslevel=args.level, **ST.seek_kw(args.seek_table), **kw)
            print("Layer zip: %s, %.1f MB from %d tarballs and %d wheels (%.1f MB), %d entries; %d bodies copied, %d "
                  "entries cleaned up; %d shared objects stripped (%d via host strip), %.1f MB -> %.1f MB"
                  % (args.dst, st["zip_bytes"] / 1e6, len(args.srcs), len(args.wheel), st["src_bytes"] / 1e6,
                     st["entries"], st["copied"]["members"], st["removed"]["entries"], st["gpu"] + st["fallback"],
                     st["fallback"], st["in_bytes"] / 1e6, st["out_bytes"] / 1e6))
        else:
            if args.keep_tests:
                ap.error("--keep-tests needs --clean or --wheel")
            st = zip_tarballs(args.srcs, args.dst, prefix=args.prefix, compresslevel=args.level,
                              **ST.seek_kw(args.seek_table), **kw)
            print("Layer zip: %s, %.1f MB from %d tarballs (%.1f MB), %d entries; %d shared objects stripped (%d via "
                  "host strip), %.1f MB -> %.1f MB"
                  % (args.dst, st["zip_bytes"] / 1e6, len(args.srcs), st["src_bytes"] / 1e6, st["entries"],
                     st["gpu"] + st["fallback"], st["fallback"], st["in_bytes"] / 1e6, st["out_bytes"] / 1e6))
    except D.CheckFailed as e:
        print("Layer zip: %s not written" % args.dst)
        print(D.summary(e.report))
        return 1
    except (OSError, ValueError, zipfile.BadZipFile) as e:
        if not args.check:
            raise
        print("error: %s" % e, file=sys.stderr)
        return 2
    if args.check:
        print(D.summary(st["check"]))
    return 0


if __name__ == "__main__":
    sys.exit(main())
