"""Drop-in installation: make an installed `lambdipy` use the CUDA strip path, CLI unchanged.

    import lambdipy_b200.patch; lambdipy_b200.patch.apply()      # or: python -m lambdipy_b200.patch build ...

Only `install_non_resolved_requirements` is replaced -- in lambdipy.project_build and in
lambdipy.cli, which imported the name (/root/reference/lambdipy/cli.py:11-16).  `lambdipy build`,
its options, PackageBuild and every other function keep running the reference's own code.

With LAMBDIPY_TARBALL_BACKEND=b200 (default: python, the reference's own code),
PackageBuild.create_compressed_tarball is replaced as well, by the mirror in tarball.py that compresses
on the GPU.  With LAMBDIPY_UNTAR_BACKEND=b200 (default: python), lambdipy.project_build.prepare_tarfile is
replaced by the mirror that inflates on the GPU (download_and_prepare_asset looks the name up at call time).

With LAMBDIPY_BUNDLE_ZIP=<path>.zip (default: unset, nothing changes), `copy_include_paths` in lambdipy.cli -- the
last step of `lambdipy build` -- is wrapped: after the reference's copy, ./build is zipped on the GPU into <path>
(zipfile_gpu.zip_tree, the archive shutil.make_archive writes) and one line reports the zip against Lambda's 50 MB
direct-upload limit and the tree against its 250 MB unzipped limit.

With LAMBDIPY_BUNDLE_VERIFY=1 (default: unset, nothing changes) and LAMBDIPY_BUNDLE_ZIP set, the written bundle is
read back on the GPU (zipfile_gpu.testzip: every member inflated and CRC-checked) before the size line; a bad member
fails the build, and the line gains the member count.  No other value is accepted.

With LAMBDIPY_BUNDLE_CHECK_DEPS=1 (default: unset, nothing changes) and LAMBDIPY_BUNDLE_ZIP set, the written bundle's
shared objects are checked on the GPU for what they need at load time (deps.check_zip at /var/task: every DT_NEEDED
found in the bundle or the runtime, the architecture, the symbol versions) after the zip and after
LAMBDIPY_BUNDLE_VERIFY's read-back; a problem fails the build, and the size line gains the count of objects checked.
No other value is accepted.

With LAMBDIPY_DEFLATE_LEVEL=9 (default: unset, the default encoder) the GPU tarball mirror and the bundle zip use
the thorough encoder (an optimal parse; smaller output, longer kernels).  No other value is accepted.

With LAMBDIPY_SEEK_TABLE=1 (default: unset, nothing changes) the GPU tarball mirror appends a seek table to the
package tarball (tarball.GpuGzipFile) and the bundle zip gives its members seek tables (zipfile_gpu.zip_tree), so
that every later read on the GPU -- the extraction of the tarball, LAMBDIPY_BUNDLE_VERIFY's read-back of the bundle --
decodes them without searching for block starts.  No other value is accepted.
"""
import os
import sys
import zipfile

TARBALL_BACKENDS = ("python", "b200")
UNTAR_BACKENDS = ("python", "b200")
LAMBDA_ZIPPED_LIMIT = 50 * 1024 * 1024  # a deployment package uploaded directly, not through S3


def bundle_zip_path():
    """LAMBDIPY_BUNDLE_ZIP, checked: None when unset, else a path ending in ".zip" that is not a directory."""
    path = os.environ.get("LAMBDIPY_BUNDLE_ZIP")
    if path is None:
        return None
    if not path.endswith(".zip") or not os.path.basename(path)[:-4] or os.path.isdir(path):
        raise ValueError("LAMBDIPY_BUNDLE_ZIP=%r: expected the path of a .zip file to write" % path)
    return path


def deflate_level():
    """LAMBDIPY_DEFLATE_LEVEL, checked: None when unset, else 9."""
    level = os.environ.get("LAMBDIPY_DEFLATE_LEVEL")
    if level is None:
        return None
    if level != "9":
        raise ValueError("LAMBDIPY_DEFLATE_LEVEL=%r: expected 9 (the optimal parse) or unset (the default encoder)" % level)
    return 9


def bundle_verify():
    """LAMBDIPY_BUNDLE_VERIFY, checked: False when unset, True for 1."""
    v = os.environ.get("LAMBDIPY_BUNDLE_VERIFY")
    if v is None:
        return False
    if v != "1":
        raise ValueError("LAMBDIPY_BUNDLE_VERIFY=%r: expected 1 (check the bundle zip on the GPU) or unset" % v)
    return True


def bundle_check_deps():
    """LAMBDIPY_BUNDLE_CHECK_DEPS, checked: False when unset, True for 1."""
    v = os.environ.get("LAMBDIPY_BUNDLE_CHECK_DEPS")
    if v is None:
        return False
    if v != "1":
        raise ValueError("LAMBDIPY_BUNDLE_CHECK_DEPS=%r: expected 1 (check the bundle's shared objects on the GPU) or unset" % v)
    return True


def seek_table():
    """LAMBDIPY_SEEK_TABLE, checked: False when unset, True for 1."""
    v = os.environ.get("LAMBDIPY_SEEK_TABLE")
    if v is None:
        return False
    if v != "1":
        raise ValueError("LAMBDIPY_SEEK_TABLE=%r: expected 1 (write a seek table into the package tarball) or unset" % v)
    return True


def zip_after_copy(copy_include_paths, zip_path, compresslevel=None, verify=False, seek=False, check_deps=False):
    """copy_include_paths followed by the bundle zip of its build directory, with verify its read-back check, with
    check_deps the load-time check of its shared objects (deps.check_zip), and the size line."""
    def wrapped(include_paths, build_directory="./build"):
        copy_include_paths(include_paths, build_directory)
        from . import project_build, zipfile_gpu
        from .seek_table import seek_kw
        level = {} if compresslevel is None else {"compresslevel": compresslevel}
        zipfile_gpu.zip_tree(build_directory, zip_path, **level, **seek_kw(seek))
        checked = ""
        if verify:
            bad = zipfile_gpu.testzip(zip_path)
            if bad is not None:
                raise RuntimeError("bundle zip %s: member %r does not read back (bad data, size or CRC-32)" % (zip_path, bad))
            with zipfile.ZipFile(zip_path) as zf:
                checked = "; %d members checked" % len(zf.infolist())
        if check_deps:
            from . import deps
            report = deps.check_zip(zip_path)
            if report["problems"]:
                raise RuntimeError("bundle zip %s: shared objects that will not load:\n%s" % (zip_path, deps.summary(report)))
            checked += "; %d shared objects checked" % report["stats"]["objects"]
        zipped, unzipped = os.path.getsize(zip_path), project_build.tree_bytes(build_directory)
        print("Bundle zip: %s, %.1f MB = %.0f %% of the 50 MB direct-upload limit; unzipped %.1f MB = %.0f %% of 250 MB%s"
              % (zip_path, zipped / 1e6, 100.0 * zipped / LAMBDA_ZIPPED_LIMIT, unzipped / 1e6,
                 100.0 * unzipped / project_build.LAMBDA_UNZIPPED_LIMIT, checked))
    return wrapped


def apply():
    backend = os.environ.get("LAMBDIPY_TARBALL_BACKEND", "python")  # checked before anything is rebound
    if backend not in TARBALL_BACKENDS:
        raise ValueError("LAMBDIPY_TARBALL_BACKEND=%r: expected one of %s" % (backend, ", ".join(TARBALL_BACKENDS)))
    untar = os.environ.get("LAMBDIPY_UNTAR_BACKEND", "python")
    if untar not in UNTAR_BACKENDS:
        raise ValueError("LAMBDIPY_UNTAR_BACKEND=%r: expected one of %s" % (untar, ", ".join(UNTAR_BACKENDS)))
    zip_path = bundle_zip_path()
    level = deflate_level()
    verify = bundle_verify()
    check_deps = bundle_check_deps()
    seek = seek_table()
    import lambdipy.cli as cli
    import lambdipy.project_build as ref
    from . import project_build as mine
    ref.install_non_resolved_requirements = mine.install_non_resolved_requirements
    cli.install_non_resolved_requirements = mine.install_non_resolved_requirements
    if backend == "b200":
        import lambdipy.package_build as ref_pkg
        from . import tarball
        from .seek_table import seek_kw
        ref_pkg.PackageBuild.create_compressed_tarball = tarball.tarball_method(level, **seek_kw(seek))
    if untar == "b200":
        from . import tarball
        ref.prepare_tarfile = tarball.prepare_tarfile
    if zip_path is not None:
        cli.copy_include_paths = zip_after_copy(ref.copy_include_paths, zip_path, level, verify=verify, seek=seek,
                                               check_deps=check_deps)
    # `lambdipy build` spends seconds resolving, downloading and copying packages before it reaches the
    # strip step (cli.py:52-67): create the CUDA context behind that, not in front of the strip
    if os.environ.get("LAMBDIPY_B200_EAGER_WARMUP", "1") != "0":
        try:
            mine.warmup()
        except ValueError:
            pass
    return cli


def main(argv=None):
    cli = apply()
    sys.argv = ["lambdipy"] + list(sys.argv[1:] if argv is None else argv)
    return cli.cli()


if __name__ == "__main__":
    main()
