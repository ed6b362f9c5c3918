"""CPU checks of the writers' `compresslevel` and of LAMBDIPY_DEFLATE_LEVEL: None keeps the default encoder (flags 0)
and 9 selects LB2_DEFLATE_BEST; every other value is refused before anything is allocated or rebound; the tarball
mirror and the bundle-zip hook pass the level through to their stand-ins, and leave the calls as before when it is
unset."""
import sys

import pytest

from lambdipy_b200 import _native as N
from lambdipy_b200 import tarball as T
from lambdipy_b200 import zipfile_gpu as Z

BAD = [0, 1, 6, 8, 10, -1, 9.0, "9", True, b"9"]


def test_flags_of_levels():
    assert N.deflate_flags(None) == 0
    assert N.deflate_flags(9) == N.DEFLATE_BEST == 1
    for bad in BAD:
        with pytest.raises(ValueError, match="compresslevel"):
            N.deflate_flags(bad)


class _NoCtx:
    """a context whose every use fails the test: a refused level must not get that far"""

    def __getattr__(self, name):
        raise AssertionError("context used (%s) before the level was checked" % name)


@pytest.mark.parametrize("bad", BAD)
def test_writers_refuse_levels_before_allocating(tmp_path, bad):
    with pytest.raises(ValueError, match="compresslevel"):
        T.GpuGzipFile(str(tmp_path / "x.gz"), ctx=_NoCtx(), compresslevel=bad)
    with pytest.raises(ValueError, match="compresslevel"):
        Z.GpuZipEncoder(_NoCtx(), compresslevel=bad)
    with pytest.raises(ValueError, match="compresslevel"):
        Z.zip_tree(str(tmp_path), str(tmp_path / "x.zip"), ctx=_NoCtx(), compresslevel=bad)
    with pytest.raises(ValueError, match="compresslevel"):
        T.gzip_tarball([], str(tmp_path / "x.tar.gz"), ctx=_NoCtx(), compresslevel=bad)
    assert not (tmp_path / "x.gz").exists() and not (tmp_path / "x.zip").exists()


class _PackageBuild:
    def __init__(self, build_dir):
        self._b = build_dir

    def git_tag(self):
        return "pkg-1.0-2"

    def build_directory(self):
        return self._b


def test_mirror_passes_the_level(tmp_path, monkeypatch):
    build = tmp_path / "build"
    (build / "pkg").mkdir(parents=True)
    monkeypatch.setenv("HOME", str(tmp_path))
    calls = []
    monkeypatch.setattr(T, "gzip_tarball", lambda srcs, path, ctx=None, **kw: calls.append(kw) or path)
    T.create_compressed_tarball(_PackageBuild(str(build)))
    T.create_compressed_tarball(_PackageBuild(str(build)), compresslevel=9)
    T.tarball_method(9)(_PackageBuild(str(build)))
    assert calls == [{}, {"compresslevel": 9}, {"compresslevel": 9}]
    assert T.tarball_method(None) is T.create_compressed_tarball
    with pytest.raises(ValueError):
        T.tarball_method(6)


@pytest.fixture
def standin(tmp_path, monkeypatch):
    pkg = tmp_path / "site" / "lambdipy"
    pkg.mkdir(parents=True)
    (pkg / "__init__.py").write_text("")
    (pkg / "project_build.py").write_text(
        "def install_non_resolved_requirements(*a, **k):\n    pass\n"
        "def copy_include_paths(include_paths, build_directory='./build'):\n    COPIED.append(build_directory)\n"
        "COPIED = []\n")
    (pkg / "cli.py").write_text("from .project_build import install_non_resolved_requirements, copy_include_paths\n")
    (pkg / "package_build.py").write_text("class PackageBuild:\n    def create_compressed_tarball(self):\n        return 'ref'\n"
                                          "    def git_tag(self):\n        return 'p-1-1'\n"
                                          "    def build_directory(self):\n        return BUILD\n")
    for k in [k for k in sys.modules if k == "lambdipy" or k.startswith("lambdipy.")]:
        monkeypatch.delitem(sys.modules, k)
    monkeypatch.syspath_prepend(str(tmp_path / "site"))
    monkeypatch.setenv("LAMBDIPY_B200_EAGER_WARMUP", "0")
    for v in ("LAMBDIPY_TARBALL_BACKEND", "LAMBDIPY_UNTAR_BACKEND", "LAMBDIPY_BUNDLE_ZIP", "LAMBDIPY_DEFLATE_LEVEL"):
        monkeypatch.delenv(v, raising=False)
    yield
    for k in [k for k in sys.modules if k == "lambdipy" or k.startswith("lambdipy.")]:
        del sys.modules[k]


@pytest.mark.parametrize("bad", ["", "6", "1", "best", "09", " 9", "9.0"])
def test_level_refused_before_rebinding(standin, monkeypatch, tmp_path, bad):
    monkeypatch.setenv("LAMBDIPY_DEFLATE_LEVEL", bad)
    monkeypatch.setenv("LAMBDIPY_TARBALL_BACKEND", "b200")
    monkeypatch.setenv("LAMBDIPY_BUNDLE_ZIP", str(tmp_path / "b.zip"))
    import lambdipy.cli as cli
    import lambdipy.package_build as ref_pkg
    import lambdipy.project_build as ref
    from lambdipy_b200 import patch
    before = (ref.install_non_resolved_requirements, cli.copy_include_paths, ref_pkg.PackageBuild.create_compressed_tarball)
    with pytest.raises(ValueError, match="LAMBDIPY_DEFLATE_LEVEL"):
        patch.apply()
    assert (ref.install_non_resolved_requirements, cli.copy_include_paths,
            ref_pkg.PackageBuild.create_compressed_tarball) == before


def test_both_hooks_pass_the_level(standin, monkeypatch, tmp_path, capsys):
    import lambdipy.cli as cli
    import lambdipy.package_build as ref_pkg
    from lambdipy_b200 import patch
    zips, tars = [], []
    monkeypatch.setattr(Z, "zip_tree", lambda root, path, ctx=None, **kw: zips.append(kw) or
                        open(path, "wb").write(b"x" * 10) and {"zip_bytes": 10})
    monkeypatch.setattr(T, "gzip_tarball", lambda srcs, path, ctx=None, **kw: tars.append(kw) or path)
    monkeypatch.setenv("HOME", str(tmp_path))
    monkeypatch.setattr(ref_pkg, "BUILD", str(tmp_path / "build"), raising=False)
    (tmp_path / "build").mkdir()
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("LAMBDIPY_TARBALL_BACKEND", "b200")
    monkeypatch.setenv("LAMBDIPY_BUNDLE_ZIP", str(tmp_path / "bundle.zip"))
    for level, kw in ((None, {}), ("9", {"compresslevel": 9})):
        if level is None:
            monkeypatch.delenv("LAMBDIPY_DEFLATE_LEVEL", raising=False)
        else:
            monkeypatch.setenv("LAMBDIPY_DEFLATE_LEVEL", level)
        patch.apply()
        ref_pkg.PackageBuild().create_compressed_tarball()
        cli.copy_include_paths(())
        assert zips[-1] == kw and tars[-1] == kw
    capsys.readouterr()
