import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu on a GPU machine")


@pytest.fixture(scope="session")
def fixture_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("elf_fixtures"))


@pytest.fixture(scope="session")
def variants(fixture_dir):
    import elf_fixtures
    v = elf_fixtures.build_variants(fixture_dir)
    assert len(v) >= 20, "toolchain built too few fixture variants: %s" % sorted(v)
    return v


@pytest.fixture(scope="session")
def note_files(fixture_dir, variants):
    import elf_fixtures
    out = {}
    for name, notes in elf_fixtures.note_scenarios().items():
        dst = os.path.join(fixture_dir, name + ".so")
        if elf_fixtures.with_build_notes(variants["c_g"], dst, notes):
            out[name] = dst
    assert out
    return out


@pytest.fixture(scope="session")
def doctored(fixture_dir, variants):
    import elf_fixtures
    return elf_fixtures.doctored(variants["c_g"], fixture_dir)


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib
    return oracle_lib.load()


@pytest.fixture(scope="session")
def gpu_ctx():
    from lambdipy_b200 import _native
    ctx = _native.Context(0)
    yield ctx
    ctx.close()
