"""CPU-side checks of the tarball path: the gzip header GpuGzipFile writes is gzip.GzipFile's, the mirror of
PackageBuild.create_compressed_tarball keeps the reference's path and add loop, and patch.apply() replaces the
method only when LAMBDIPY_TARBALL_BACKEND=b200 (lambdipy.package_build is not even imported otherwise)."""
import glob
import gzip
import io
import os
import sys

import pytest


@pytest.mark.parametrize("name", ["pkg-1.0-1.tar.gz", "/home/u/.lambdipy/build/numpy-1.19.5-2.tar.gz", "plain.tar",
                                  "café.tar.gz", "中.tar.gz", b"/tmp/bytes-name.tar.gz"])
def test_gzip_header_equals_stdlib(name):
    from lambdipy_b200.tarball import gzip_header
    buf = io.BytesIO()
    with gzip.GzipFile(filename=name, mode="wb", compresslevel=9, fileobj=buf, mtime=1234567890):
        pass
    mine = gzip_header(name, 1234567890)
    assert buf.getvalue()[:len(mine)] == mine
    assert buf.getvalue()[len(mine):] == b"\x03\x00" + b"\0" * 8   # nothing of the header is left over


class _PackageBuild:
    def __init__(self, build_dir):
        self._dir = build_dir

    def git_tag(self):
        return "pkg-1.0-2"

    def build_directory(self):
        return self._dir


def test_mirror_path_and_sources(tmp_path, monkeypatch):
    from lambdipy_b200 import tarball
    build = tmp_path / "build" / "pkg" / "1.0"
    (build / "pkg").mkdir(parents=True)
    (build / "pkg.libs").mkdir()
    (build / "top.py").write_text("x = 1\n")
    (build / ".hidden").write_text("")   # glob's "*" skips dot files, as in the reference
    monkeypatch.setenv("HOME", str(tmp_path))
    calls = []
    monkeypatch.setattr(tarball, "gzip_tarball", lambda srcs, path, ctx=None: calls.append((list(srcs), path)) or path)
    path = tarball.create_compressed_tarball(_PackageBuild(str(build)))
    assert path == "%s/.lambdipy/build/pkg-1.0-2.tar.gz" % tmp_path
    assert calls == [(glob.glob("%s/*" % build), path)]
    assert sorted(os.path.basename(p) for p in calls[0][0]) == ["pkg", "pkg.libs", "top.py"]


@pytest.fixture
def standin_lambdipy(tmp_path, monkeypatch):
    pkg = tmp_path / "site" / "lambdipy"
    pkg.mkdir(parents=True)
    (pkg / "__init__.py").write_text("")
    (pkg / "project_build.py").write_text("def install_non_resolved_requirements(*a, **k):\n    raise AssertionError\n")
    (pkg / "cli.py").write_text("from .project_build import install_non_resolved_requirements\n")
    (pkg / "package_build.py").write_text("class PackageBuild:\n    def create_compressed_tarball(self):\n        return 'ref'\n")
    for k in [k for k in sys.modules if k == "lambdipy" or k.startswith("lambdipy.")]:
        monkeypatch.delitem(sys.modules, k)
    monkeypatch.syspath_prepend(str(tmp_path / "site"))
    monkeypatch.setenv("LAMBDIPY_B200_EAGER_WARMUP", "0")
    yield
    for k in [k for k in sys.modules if k == "lambdipy" or k.startswith("lambdipy.")]:
        del sys.modules[k]


def test_patch_leaves_tarball_alone_by_default(standin_lambdipy, monkeypatch):
    monkeypatch.delenv("LAMBDIPY_TARBALL_BACKEND", raising=False)
    import lambdipy_b200.patch as patch
    patch.apply()
    assert "lambdipy.package_build" not in sys.modules
    import lambdipy.package_build as ref_pkg
    assert ref_pkg.PackageBuild().create_compressed_tarball() == "ref"
    monkeypatch.setenv("LAMBDIPY_TARBALL_BACKEND", "python")
    patch.apply()
    assert ref_pkg.PackageBuild().create_compressed_tarball() == "ref"


def test_patch_installs_gpu_tarball_when_asked(standin_lambdipy, monkeypatch):
    import lambdipy_b200.patch as patch
    from lambdipy_b200 import tarball
    monkeypatch.setenv("LAMBDIPY_TARBALL_BACKEND", "b200")
    patch.apply()
    import lambdipy.package_build as ref_pkg
    assert ref_pkg.PackageBuild.create_compressed_tarball is tarball.create_compressed_tarball

def test_patch_rejects_unknown_backend_before_patching(standin_lambdipy, monkeypatch):
    import lambdipy_b200.patch as patch
    import lambdipy.project_build as ref_pb
    import lambdipy.cli as cli
    before = ref_pb.install_non_resolved_requirements
    monkeypatch.setenv("LAMBDIPY_TARBALL_BACKEND", "pigz")
    with pytest.raises(ValueError):
        patch.apply()
    assert ref_pb.install_non_resolved_requirements is before and cli.install_non_resolved_requirements is before
    assert "lambdipy.package_build" not in sys.modules


def test_default_context_reuses_warmup_or_honours_device(monkeypatch):
    from lambdipy_b200 import project_build, tarball
    from lambdipy_b200 import _native as N

    class Warm:
        def result(self):
            return "warm-ctx"
    monkeypatch.setattr(project_build, "_warm", Warm())
    assert tarball._default_context() == ("warm-ctx", False)
    monkeypatch.setattr(project_build, "_warm", None)
    monkeypatch.setenv("LAMBDIPY_B200_DEVICE", "3")
    monkeypatch.setattr(N, "Context", lambda device: ("new-ctx", device))
    assert tarball._default_context() == (("new-ctx", 3), True)


def test_gzip_tarball_is_public():
    import lambdipy_b200
    from lambdipy_b200 import tarball
    assert lambdipy_b200.gzip_tarball is tarball.gzip_tarball
