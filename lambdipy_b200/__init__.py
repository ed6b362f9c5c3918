"""lambdipy_b200 -- the shared-object strip pass of customink/lambdipy on H100 (sm_90a).

Public surface:
    strip_tree(build_directory)                 replaces `find ... -name "*.so" | xargs strip`
                                                (/root/reference/lambdipy/project_build.py:260)
    strip_buffers(ctx, [bytes, ...])            same operation on in-memory ELF images
    project_build.install_non_resolved_requirements   mirror of the reference entry point
    gzip_tarball(src_paths, tarball_path)       tar.gz of a package tree, DEFLATE on the GPU
    tarball.create_compressed_tarball           mirror of PackageBuild.create_compressed_tarball
    gunzip(path)                                decompressed bytes of a gzip file, DEFLATE decoded on the GPU
    strip_tarball(src, dst)                     a .tar.gz with its shared objects stripped, inflated, stripped
                                                and deflated on the GPU without unpacking it
    tarball.prepare_tarfile                     mirror of the reference's prepare_tarfile
    zip_tree(root_dir, zip_path)                the Lambda deployment zip of a tree (shutil.make_archive's
                                                archive), every member's DEFLATE body compressed on the GPU
    extract_zip(zip_path, directory)            ZipFile.extractall's tree, every member inflated on the GPU
    testzip(zip_path)                           ZipFile.testzip's answer, every member checked on the GPU
    zip_tarballs(srcs, dst, prefix="")          the Lambda zip of .tar.gz package assets, shared objects stripped,
                                                inflated, stripped and deflated on the GPU without unpacking them
    zip_build(dst, tarballs, wheels)            the Lambda zip of a whole build: tarballs and wheels, pip's target
                                                install and the build script's clean-up restated, strip on the GPU
    check_zip(zip_path, mount="/var/task")      whether the zip's shared objects will load on Lambda: dynamic
                                                sections read on the GPU, the loader's search restated
    patch.apply()                               monkey-patch an installed lambdipy in place
The byte work is done by liblambdipy_b200.so (CUDA, C ABI in include/lambdipy_b200.h).
"""
__version__ = "0.1.0"


def __getattr__(name):
    if name in ("strip_tree", "strip_buffers"):
        from . import strip
        return getattr(strip, name)
    if name in ("gzip_tarball", "gunzip", "strip_tarball"):
        from . import tarball
        return getattr(tarball, name)
    if name in ("zip_tree", "extract_zip", "testzip"):
        from . import zipfile_gpu
        return getattr(zipfile_gpu, name)
    if name in ("zip_tarballs", "zip_build"):
        from . import layer
        return getattr(layer, name)
    if name == "check_zip":
        from . import deps
        return deps.check_zip
    raise AttributeError(name)
