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
"""
import os
import posixpath
import stat
import sys
import tempfile
import time
import zipfile

from . import _native as N
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
    return sorted(chosen.values(), key=lambda f: (f.src, f.member.offset_data)), skipped


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
             tolerate_non_elf=False):
    """zip_tarballs with the engines given (tarball.GpuTarReader, tarball.GpuTarIndex, zipfile_gpu.GpuStripper,
    zipfile_gpu.GpuZipEncoder fed by submit_device, or stand-ins with the same interfaces)."""
    srcs = [os.fspath(srcs)] if isinstance(srcs, (str, bytes, os.PathLike)) else [os.fspath(s) for s in srcs]
    dst = os.fspath(dst)
    check_prefix(prefix)
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
    return st


def zip_tarballs(srcs, dst, prefix="", ctx=None, compresslevel=None, fallback_host_strip=True, tolerate_non_elf=False,
                 piece_bytes=PIECE_BYTES, seek_table=False):
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
    index, inflate, strip and deflate (the engines' stats) and kernel_ms, their kernel times summed.  There is no CPU
    path: without a GPU this raises."""
    N.deflate_flags(compresslevel)
    check_prefix(prefix)
    own = False
    if ctx is None:
        ctx, own = T._default_context()
    try:
        with T.GpuTarReader(ctx) as reader, Z.GpuStripper(ctx) as stripper, \
                Z.GpuZipEncoder(ctx, piece_bytes, compresslevel=compresslevel, host_buffers=False,
                                seek_table=seek_table) as enc:
            return zip_with(srcs, dst, reader, T.GpuTarIndex(ctx), stripper, enc, prefix, fallback_host_strip,
                            tolerate_non_elf)
    finally:
        if own:
            ctx.close()


def main(argv=None):
    """python -m lambdipy_b200.layer DST SRC [SRC ...] [--prefix python/] [--level 9] [--seek-table]"""
    import argparse
    ap = argparse.ArgumentParser(prog="python -m lambdipy_b200.layer",
                                 description="write the Lambda zip of .tar.gz package assets, shared objects stripped, "
                                             "inflated, stripped and deflated on the GPU")
    ap.add_argument("dst")
    ap.add_argument("srcs", nargs="+", metavar="src")
    ap.add_argument("--prefix", default="", help='directory of the zip the sources go under ("python/" for a layer)')
    ap.add_argument("--level", type=int, choices=[9], default=None, help="9: the optimal parse (smaller, slower)")
    ap.add_argument("--seek-table", action="store_true",
                    help="give multi-chunk members seek tables, with which the GPU reader decodes them without search")
    args = ap.parse_args(argv)
    st = zip_tarballs(args.srcs, args.dst, prefix=args.prefix, compresslevel=args.level, **ST.seek_kw(args.seek_table))
    print("Layer zip: %s, %.1f MB from %d tarballs (%.1f MB), %d entries; %d shared objects stripped (%d via host "
          "strip), %.1f MB -> %.1f MB"
          % (args.dst, st["zip_bytes"] / 1e6, len(args.srcs), st["src_bytes"] / 1e6, st["entries"],
             st["gpu"] + st["fallback"], st["fallback"], st["in_bytes"] / 1e6, st["out_bytes"] / 1e6))
    return 0


if __name__ == "__main__":
    sys.exit(main())
