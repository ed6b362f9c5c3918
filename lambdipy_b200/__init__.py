"""lambdipy_b200 -- the shared-object strip pass of customink/lambdipy on H100 (sm_90a).

Public surface:
    strip_tree(build_directory)                 replaces `find ... -name "*.so" | xargs strip`
                                                (/root/reference/lambdipy/project_build.py:260)
    strip_buffers(ctx, [bytes, ...])            same operation on in-memory ELF images
    project_build.install_non_resolved_requirements   mirror of the reference entry point
    gzip_tarball(src_paths, tarball_path)       tar.gz of a package tree, DEFLATE on the GPU
    tarball.create_compressed_tarball           mirror of PackageBuild.create_compressed_tarball
    gunzip(path)                                decompressed bytes of a gzip file, DEFLATE decoded on the GPU
    tarball.prepare_tarfile                     mirror of the reference's prepare_tarfile
    patch.apply()                               monkey-patch an installed lambdipy in place
The byte work is done by liblambdipy_b200.so (CUDA, C ABI in include/lambdipy_b200.h).
"""
__version__ = "0.1.0"


def __getattr__(name):
    if name in ("strip_tree", "strip_buffers"):
        from . import strip
        return getattr(strip, name)
    if name in ("gzip_tarball", "gunzip"):
        from . import tarball
        return getattr(tarball, name)
    raise AttributeError(name)
