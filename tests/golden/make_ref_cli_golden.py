#!/usr/bin/env python
"""Records, as tests/golden/ref_cli.json, how the REFERENCE's click CLI (lambdipy/cli.py of a checkout of
customink/lambdipy given on the command line) reaches the strip step: the names cli.py imports from
project_build, the options and parameters of its `build` command, and the call it makes to
install_non_resolved_requirements.  Only these names are stored (read with `ast`, nothing is executed);
tests/test_patch_reference_cli.py builds its stand-in CLI from them."""
import ast
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def const(node):
    return node.value if isinstance(node, ast.Constant) else None


def main():
    if len(sys.argv) != 2:
        sys.exit("usage: make_ref_cli_golden.py <checkout of customink/lambdipy>")
    tree = ast.parse(open(os.path.join(sys.argv[1], "lambdipy", "cli.py")).read())
    imports = [a.name for n in tree.body if isinstance(n, ast.ImportFrom) and n.module == "project_build" and n.level == 1
               for a in n.names]
    build = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "build")
    options = []
    for d in build.decorator_list:  # source order, top to bottom
        if isinstance(d, ast.Call) and isinstance(d.func, ast.Attribute) and d.func.attr == "option":
            kw = {k.arg: const(k.value) for k in d.keywords}
            options.append({"decls": [const(x) for x in d.args], "is_flag": bool(kw.get("is_flag")), "multiple": bool(kw.get("multiple"))})
    call = next(n for n in ast.walk(build) if isinstance(n, ast.Call) and isinstance(n.func, ast.Name)
                and n.func.id == "install_non_resolved_requirements")
    record = {
        "source": "lambdipy/cli.py of customink/lambdipy",
        "imports_from_project_build": imports,
        "build_command": {"params": [a.arg for a in build.args.args], "options": options},
        "strip_step_call": {"function": "install_non_resolved_requirements", "args": [a.id for a in call.args],
                            "keywords": [k.arg for k in call.keywords]},
    }
    with open(os.path.join(HERE, "ref_cli.json"), "w") as f:
        json.dump(record, f, indent=1)
        f.write("\n")
    print(json.dumps(record, indent=1))


if __name__ == "__main__":
    main()
