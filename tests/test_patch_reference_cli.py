"""Drop-in check at the CLI level: lambdipy_b200.patch.apply() rebinds install_non_resolved_requirements
in lambdipy.project_build and in lambdipy.cli (which imported the name), so `lambdipy build --no-docker`
runs our mirror.  The installed lambdipy is represented by a stand-in package generated from a record of
the reference's own cli.py (tests/golden/ref_cli.json, made by tests/golden/make_ref_cli_golden.py): the
same names imported from project_build, a click `build` command with the same options, and the same
positional call of install_non_resolved_requirements."""
import inspect
import json
import os
import shutil
import sys

import pytest

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ref_cli.json")


def _standin_sources(rec):
    names = rec["imports_from_project_build"]
    pb = ["class %s(Exception):\n    pass\n" % n if n[0].isupper() else
          "def %s(*args, **kwargs):\n    raise AssertionError('stand-in %s ran: not expected in this test')\n" % (n, n)
          for n in names]
    opts = "".join("@click.option(%s, is_flag=%r, multiple=%r)\n" % (", ".join(repr(d) for d in o["decls"]), o["is_flag"], o["multiple"])
                   for o in rec["build_command"]["options"])
    call = rec["strip_step_call"]
    cli = ("import click\n"
           "from .project_build import %s\n\n\n"
           "@click.group()\n"
           "def cli():\n    pass\n\n\n"
           "@cli.command()\n%s"
           "def build(%s):\n"
           "    resolved_requirements, requirements, python_version = {}, [], '3.7'\n"
           "    %s(%s)\n"
           "    print('Build done')\n") % (", ".join(names), opts, ", ".join(rec["build_command"]["params"]),
                                         call["function"], ", ".join(call["args"]))
    return "\n".join(pb), cli


@pytest.fixture
def record():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.fixture
def standin_lambdipy(record, tmp_path, monkeypatch):
    pkg = tmp_path / "site" / "lambdipy"
    pkg.mkdir(parents=True)
    pb, cli = _standin_sources(record)
    (pkg / "__init__.py").write_text("")
    (pkg / "project_build.py").write_text(pb)
    (pkg / "cli.py").write_text(cli)
    for k in [k for k in sys.modules if k == "lambdipy" or k.startswith("lambdipy.")]:
        monkeypatch.delitem(sys.modules, k)
    monkeypatch.syspath_prepend(str(tmp_path / "site"))
    yield
    for k in [k for k in sys.modules if k == "lambdipy" or k.startswith("lambdipy.")]:
        del sys.modules[k]


def test_mirror_signature_matches_reference_call(record):
    """the reference CLI imports the name patch.apply() rebinds and calls it positionally in the mirror's parameter order"""
    from lambdipy_b200 import project_build as mine
    call = record["strip_step_call"]
    assert call["function"] in record["imports_from_project_build"]
    params = list(inspect.signature(mine.install_non_resolved_requirements).parameters)
    assert params[:len(call["args"])] == call["args"] and not call["keywords"]
    assert any("--no-docker" in o["decls"] and o["is_flag"] for o in record["build_command"]["options"])


def test_patched_cli_build_runs_our_strip_step(standin_lambdipy, tmp_path, monkeypatch, variants):
    click_testing = pytest.importorskip("click.testing")
    monkeypatch.setenv("LAMBDIPY_B200_EAGER_WARMUP", "0")
    import lambdipy_b200.patch as patch
    cli = patch.apply()
    import lambdipy.project_build as ref_pb
    from lambdipy_b200 import project_build as mine
    assert ref_pb.install_non_resolved_requirements is mine.install_non_resolved_requirements
    assert cli.install_non_resolved_requirements is mine.install_non_resolved_requirements

    work = tmp_path / "proj"
    (work / "build").mkdir(parents=True)
    monkeypatch.chdir(work)
    monkeypatch.setenv("LAMBDIPY_STRIP_BACKEND", "gnu")       # the reference's own line as backend: no GPU needed
    # an empty tree makes the reference's line fail (xargs runs `strip` without arguments, rc 123)
    r = click_testing.CliRunner().invoke(cli.cli, ["build", "--no-docker"])
    assert r.exit_code == 123, r.output
    shutil.copy(variants["c_g"], os.path.join("build", "mod.so"))
    before = os.path.getsize(variants["c_g"])
    r = click_testing.CliRunner().invoke(cli.cli, ["build", "--no-docker"])
    assert r.exit_code == 0, r.output
    assert "Finalizing the build" in r.output and "Build done" in r.output
    assert os.path.getsize(work / "build" / "mod.so") < before      # stripped by the (gnu) backend of our mirror
    assert not (work / "build" / "build").exists()
