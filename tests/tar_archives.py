"""Tar streams for the tar walk and strip_tarball tests: tarfile's and GNU tar's formats, long and non-ASCII names,
pax records, base-256 sizes, sparse members, a directory header with a size, trailing garbage, truncation and a bad
checksum.  Every archive is built from a seed or from fixed bytes, so a failure names one reproducible stream."""
import io
import os
import shutil
import subprocess
import tarfile


def tree(root, files):
    """files: {relative path: bytes, or ("sym", target), or ("dir",)}"""
    for name, what in files.items():
        p = os.path.join(root, name)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        if isinstance(what, bytes):
            with open(p, "wb") as f:
                f.write(what)
        elif what[0] == "sym":
            os.symlink(what[1], p)
        else:
            os.makedirs(p, exist_ok=True)
    return root


def sample_tree(root):
    long_dir = "d" * 60 + "/" + "e" * 60
    return tree(root, {
        "pkg/__init__.py": b"",
        "pkg/mod.py": b"print('hello')\n" * 40,
        "pkg/lib/libx.so.1": b"\x7fELF" + bytes(range(256)) * 9,
        "pkg/lib/libx.so": ("sym", "libx.so.1"),
        "pkg/" + long_dir + "/deep_" + "n" * 90 + ".so": b"\x7fELF deep" * 70,
        "pkg/näme_ünicode.txt": b"umlauts\n",
        "pkg/link_" + "l" * 120 + ".so": ("sym", "lib/libx.so.1"),
        "pkg/empty": ("dir",),
        "pkg/zero.bin": b"",
    })


def tarfile_bytes(root, fmt, **kw):
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=fmt, **kw) as tar:
        tar.add(root, arcname=os.path.basename(root))
    return buf.getvalue()


def gnu_tar_bytes(root, fmt, tmp, *extra):
    """GNU tar's output in one of its formats; None where GNU tar is missing or refuses the tree in that format"""
    if not shutil.which("tar"):
        return None
    out = os.path.join(tmp, "gnu_%s.tar" % fmt)
    r = subprocess.run(["tar", "--format=" + fmt, *extra, "-cf", out, "-C", os.path.dirname(root), os.path.basename(root)],
                       capture_output=True)
    if r.returncode != 0:
        return None
    with open(out, "rb") as f:
        return f.read()


def seal(block):
    """a header block with its checksum recomputed"""
    b = bytearray(block)
    b[148:156] = b"%06o\0 " % tarfile.calc_chksums(bytes(b))[0]
    return bytes(b)


def crafted():
    """archives whose headers no writer produces on its own: {name: bytes}"""
    out = {}
    # a pax size record that disagrees with the ustar size field: tarfile follows the record
    ti = tarfile.TarInfo("pax/size_record.so")
    data = b"\x7fELF" + b"p" * 3000
    ti.size = len(data)
    ti.pax_headers = {"size": str(len(data))}
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.PAX_FORMAT) as tar:
        tar.addfile(ti, io.BytesIO(data))
        tar.addfile(tarfile.TarInfo("pax/after.txt"), io.BytesIO(b""))
    raw = bytearray(buf.getvalue())
    pax_len = 512 + -(-tarfile.nti(raw[124:136]) // 512) * 512
    hdr = bytearray(raw[pax_len:pax_len + 512])
    hdr[124:136] = tarfile.itn(0, 12, tarfile.USTAR_FORMAT)
    raw[pax_len:pax_len + 512] = seal(hdr)
    out["pax_size_record"] = bytes(raw)
    # base-256 size fields (GNU), on a small member
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.GNU_FORMAT) as tar:
        for name, n in (("b256/a.so", 1500), ("b256/b.txt", 10)):
            ti = tarfile.TarInfo(name)
            ti.size = n
            tar.addfile(ti, io.BytesIO(b"\x7fELF" + b"b" * (n - 4) if n > 4 else b"x" * n))
    raw = bytearray(buf.getvalue())
    for off in (0, 512 + 1536):
        h = bytearray(raw[off:off + 512])
        n = tarfile.nti(h[124:136])
        h[124:136] = bytes([0x80]) + n.to_bytes(11, "big")
        raw[off:off + 512] = seal(h)
    out["base256_sizes"] = bytes(raw)
    # a directory header with a non-zero size: tarfile does not skip it
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.GNU_FORMAT) as tar:
        d = tarfile.TarInfo("sized_dir.so")
        d.type, d.size = tarfile.DIRTYPE, 4096
        tar.addfile(d)
        tar.addfile(tarfile.TarInfo("sized_dir.so/x.txt"), io.BytesIO(b""))
        f = tarfile.TarInfo("sized_dir.so/y.so")
        f.size = 700
        tar.addfile(f, io.BytesIO(b"\x7fELF" + b"y" * 696))
    out["dir_with_size"] = buf.getvalue()
    # a global pax header in front of the members
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.PAX_FORMAT, pax_headers={"comment": "global"}) as tar:
        for i in range(3):
            ti = tarfile.TarInfo("g/%d.so" % i)
            ti.size = 600 * (i + 1)
            tar.addfile(ti, io.BytesIO(b"\x7fELF" + bytes(ti.size - 4)))
    out["pax_global"] = buf.getvalue()
    # v7-style: AREGTYPE directory entry ending in '/', and an AREGTYPE file
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.USTAR_FORMAT) as tar:
        d = tarfile.TarInfo("v7dir/")
        d.type, d.size = tarfile.AREGTYPE, 1024
        tar.addfile(d)
        f = tarfile.TarInfo("v7dir/f.so")
        f.type, f.size = tarfile.AREGTYPE, 100
        tar.addfile(f, io.BytesIO(b"\x7fELF" + bytes(96)))
    out["v7_aregtype"] = buf.getvalue()
    return out


def damaged(good):
    """variants of a good archive: {name: bytes}"""
    members = tarfile.open(fileobj=io.BytesIO(good)).getmembers()
    last = members[-1]
    bad = bytearray(good)
    bad[last.offset + 10] ^= 0x55                 # the last header's checksum no longer matches
    mid = members[len(members) // 2]
    return {
        "trailing_garbage": good + bytes(range(256)) * 7,
        "bad_checksum": bytes(bad),
        "truncated_in_header": good[:last.offset + 300],
        "truncated_in_data": good[:members[1].offset_data + 10] if members[1].size > 10 else good[:members[1].offset + 100],
        "no_end_marker": good[:mid.offset],
        "empty": b"",
    }
