#!/usr/bin/env python
"""Runs the REFERENCE's own install_non_resolved_requirements (imported from a checkout of
customink/lambdipy given on the command line, its missing third-party imports stubbed) on a scratch
tree and records (a) the script it generates and (b) the file list / sizes after its strip, as
tests/golden/ref_script.json.  The tests check the mirror in lambdipy_b200/project_build.py against
this record, so they do not need the reference."""
import contextlib
import io
import json
import os
import shutil
import sys
import tempfile
import types

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import elf_fixtures as F  # noqa: E402

for name in ("docker", "requirementslib", "github", "github.GithubException", "github.GitRelease"):
    m = types.ModuleType(name)
    m.Requirement = object
    m.Github = object
    m.InputGitAuthor = object
    m.UnknownObjectException = Exception
    m.GitRelease = object
    sys.modules[name] = m
if len(sys.argv) != 2:
    sys.exit("usage: make_ref_script_golden.py <checkout of customink/lambdipy>")
sys.path.insert(0, sys.argv[1])
from lambdipy import project_build as ref  # noqa: E402


class Req:
    def __init__(self, name):
        self.name = name


def main():
    tmp = tempfile.mkdtemp()
    v = F.build_variants(os.path.join(tmp, "fx"))
    cases = {}
    for case, keep_tests in (("default", None), ("keep_tests", ["numpy", "scipy"])):
        bd = os.path.join(tmp, "build_" + case)
        os.makedirs(os.path.join(bd, "pkg", "tests"))
        os.makedirs(os.path.join(bd, "pkg", "__pycache__"))
        os.makedirs(os.path.join(bd, "pkg-1.0.dist-info"))
        for k in ("c_g", "cxx_g", "c_gold"):
            shutil.copy(v[k], os.path.join(bd, "pkg", k + ".so"))
        shutil.copy(v["c_plain"], os.path.join(bd, "pkg", "libversioned.so.1"))  # not matched by *.so
        os.symlink("c_g.so", os.path.join(bd, "pkg", "link.so"))
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            ref.install_non_resolved_requirements({"x": object()}, [{"line": "x==1", "requirement": Req("x")}], "3.12",
                                                  keep_tests=keep_tests, no_docker=True, build_directory=bd)
        listing = {}
        for d, dirs, fs in os.walk(bd):
            for f in fs + dirs:
                p = os.path.join(d, f)
                listing[os.path.relpath(p, bd)] = "link" if os.path.islink(p) else ("dir" if os.path.isdir(p) else os.path.getsize(p))
        cases[case] = {"stdout": out.getvalue().replace(bd, "{BUILD}"), "listing": listing,
                       "inputs": {k: os.path.getsize(v[k]) for k in ("c_g", "cxx_g", "c_gold", "c_plain")}}
    with open(os.path.join(HERE, "ref_script.json"), "w") as f:
        json.dump(cases, f, indent=1, sort_keys=True)
    print(json.dumps(cases["default"], indent=1)[:1500])
    shutil.rmtree(tmp)


if __name__ == "__main__":
    main()
