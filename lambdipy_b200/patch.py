"""Drop-in installation: make an installed `lambdipy` use the CUDA strip path, CLI unchanged.

    import lambdipy_b200.patch; lambdipy_b200.patch.apply()      # or: python -m lambdipy_b200.patch build ...

Only `install_non_resolved_requirements` is replaced -- in lambdipy.project_build and in
lambdipy.cli, which imported the name (/root/reference/lambdipy/cli.py:11-16).  `lambdipy build`,
its options, PackageBuild and every other function keep running the reference's own code.

With LAMBDIPY_TARBALL_BACKEND=b200 (default: python, the reference's own code),
PackageBuild.create_compressed_tarball is replaced as well, by the mirror in tarball.py that compresses
on the GPU.  With LAMBDIPY_UNTAR_BACKEND=b200 (default: python), lambdipy.project_build.prepare_tarfile is
replaced by the mirror that inflates on the GPU (download_and_prepare_asset looks the name up at call time).
"""
import os
import sys

TARBALL_BACKENDS = ("python", "b200")
UNTAR_BACKENDS = ("python", "b200")


def apply():
    backend = os.environ.get("LAMBDIPY_TARBALL_BACKEND", "python")  # checked before anything is rebound
    if backend not in TARBALL_BACKENDS:
        raise ValueError("LAMBDIPY_TARBALL_BACKEND=%r: expected one of %s" % (backend, ", ".join(TARBALL_BACKENDS)))
    untar = os.environ.get("LAMBDIPY_UNTAR_BACKEND", "python")
    if untar not in UNTAR_BACKENDS:
        raise ValueError("LAMBDIPY_UNTAR_BACKEND=%r: expected one of %s" % (untar, ", ".join(UNTAR_BACKENDS)))
    import lambdipy.cli as cli
    import lambdipy.project_build as ref
    from . import project_build as mine
    ref.install_non_resolved_requirements = mine.install_non_resolved_requirements
    cli.install_non_resolved_requirements = mine.install_non_resolved_requirements
    if backend == "b200":
        import lambdipy.package_build as ref_pkg
        from . import tarball
        ref_pkg.PackageBuild.create_compressed_tarball = tarball.create_compressed_tarball
    if untar == "b200":
        from . import tarball
        ref.prepare_tarfile = tarball.prepare_tarfile
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
