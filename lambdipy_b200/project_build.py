"""Host-side mirror of the one reference entry point that contains the strip step.

Reference: lambdipy.project_build.install_non_resolved_requirements
(/root/reference/lambdipy/project_build.py:234-277).  That function writes a bash script into
`<build_directory>/build` -- pip install of the unresolved requirements, removal of *.egg-info,
*.dist-info, __pycache__ and tests directories, and, last, `find ... -name "*.so" | xargs strip`
(:260) -- runs it on the host (:268) or in a lambci container (:274) and deletes it (:277).

This mirror keeps the signature, the printed messages, the script (minus its last line) and the
exit-code convention, and performs the strip with the CUDA library on the build tree once the
script has finished.  Nothing else of the reference is re-implemented here: requirement
resolution, Docker builds, release download stay in the reference package (see patch.py).

Backend switch (additive; the reference's TODO at cli.py:34-39 asks for one):
    LAMBDIPY_STRIP_BACKEND=b200   default: CUDA path; raises if no H100 / library is present
    LAMBDIPY_STRIP_BACKEND=gnu    the reference's own shell line, untouched
    LAMBDIPY_STRIP_BACKEND=off    do not strip
"""
import os
import stat
import subprocess
import sys
import threading

XARGS_FAILURE_RC = 123  # what `find | xargs strip` returns when any strip invocation fails


def _backend(backend=None):
    backend = (backend or os.environ.get("LAMBDIPY_STRIP_BACKEND", "b200")).lower()
    if backend not in ("b200", "gnu", "off"):
        raise ValueError("LAMBDIPY_STRIP_BACKEND must be b200, gnu or off (got %r)" % backend)
    return backend


def _keep_pattern(keep_tests):
    return "\\|".join(keep_tests) if keep_tests else "*"  # project_build.py:249


def _script_lines(install_dir, pip_args, keep_tests, cleanup_in_script=True):
    pip_line = ("pip install %s -t %s" % (pip_args, install_dir)) if pip_args else ""
    lines = ["#!/bin/bash", "set -ex", pip_line]
    if cleanup_in_script:  # project_build.py:256-259; the b200 backend does these on its own walk
        lines += [
            "rm -rf %s/*.egg-info" % install_dir,
            "rm -rf %s/*.dist-info" % install_dir,
            "find %s/ -name __pycache__ | xargs rm -rf" % install_dir,
            'find %s/ -name tests | grep -v "%s" | xargs rm -rf' % (install_dir, _keep_pattern(keep_tests)),
        ]
    return lines


def _reference_strip_line(install_dir):
    return 'find %s/ -name "*.so" | xargs strip' % install_dir  # project_build.py:260


# ---------------------------------------------------------------- CUDA warm-up behind the script
class _Warmup:
    """Creating the CUDA context (and lb2_strip_tree's pinned slot ring, streams, workspaces) takes
    longer than stripping a small tree.  It does not depend on the tree, so it runs on a helper
    thread while the reference's script is busy with pip / rm (project_build.py:266-274)."""

    def __init__(self, device, build_directory=None):
        self.device, self.ctx, self.error, self.build_directory = device, None, None, build_directory
        self.prepared = False
        self.thread = threading.Thread(target=self._run, name="lambdipy-b200-warmup", daemon=True)
        self.thread.start()

    @staticmethod
    def _so_bytes(build_directory):
        total = 0
        for d, _, fs in os.walk(build_directory):
            for f in fs:
                if f.endswith(".so"):
                    try:
                        total += os.path.getsize(os.path.join(d, f))
                    except OSError:
                        pass
        return total

    def _prepare(self, build_directory):
        # size the pinned slot ring for what is already in the tree (prebuilt packages are copied in before this step,
        # project_build.py:169-175); pip may add more, the ring is only a staging area
        if self.ctx is not None and not self.prepared and build_directory and os.path.isdir(build_directory):
            self.ctx.check(self.ctx.lib.lb2_tree_prepare(self.ctx.h, max(self._so_bytes(build_directory), 1 << 24)))
            self.prepared = True

    def _run(self):
        try:
            from . import _native as N
            self.ctx = N.Context(self.device)
            self._prepare(self.build_directory)
        except BaseException as e:  # re-raised on the caller's thread by result()
            self.error = e

    def result(self):
        self.thread.join()
        if self.error is not None:
            raise self.error
        return self.ctx


_warm = None


def warmup(backend=None, build_directory=None):
    """Start (once) creating the CUDA context in the background; no-op for the gnu/off backends."""
    global _warm
    if _backend(backend) == "b200" and _warm is None:
        _warm = _Warmup(int(os.environ.get("LAMBDIPY_B200_DEVICE", "0")), build_directory)
    return _warm


def _context():
    w = warmup("b200")
    return w.result()  # raises ImportError / NoDeviceError: no silent CPU path


def strip_build_tree(build_directory, backend=None, cleanup=False, keep_tests=None):
    """The replacement for project_build.py:260 (and, with cleanup=True, :256-259).  Returns the
    process-style return code."""
    backend = _backend(backend)
    if backend == "off":
        return 0
    if backend == "gnu":
        return subprocess.call(["bash", "-c", "set -o pipefail; " + _reference_strip_line(build_directory)])
    from .strip import strip_tree
    st = strip_tree(build_directory, suffix=".so", fallback_host_strip=True, ctx=_context(), cleanup=cleanup,
                    keep_tests_regex=_keep_pattern(keep_tests) if cleanup else None)
    print("Stripped %d shared objects on the GPU (%d via host strip), %.1f MB -> %.1f MB" %
          (st["n_gpu"], st["n_fallback"], st["in_bytes"] / 1e6, st["out_bytes"] / 1e6))
    print(bundle_report(build_directory))
    return XARGS_FAILURE_RC if st["n_failed"] else 0


LAMBDA_UNZIPPED_LIMIT = 250 * 1024 * 1024  # the limit the reference exists to meet (/root/reference/README.md:4-5)


def tree_bytes(build_directory):
    """bytes of the regular files under build_directory (symlinks not counted)"""
    total = 0
    for d, _, fs in os.walk(build_directory):
        for f in fs:
            p = os.path.join(d, f)
            if not os.path.islink(p):
                total += os.path.getsize(p)
    return total


def bundle_report(build_directory):
    """Size of the finished bundle against Lambda's 250 MB unzipped limit (the reference's README
    promises 'tips to further improve your bundle size' as a TODO, README.md:23)."""
    total = tree_bytes(build_directory)
    pct = 100.0 * total / LAMBDA_UNZIPPED_LIMIT
    return "Bundle size: %.1f MB = %.0f %% of the 250 MB Lambda limit%s" % (total / 1e6, pct, "" if pct <= 100 else "  ** over the limit **")


def install_non_resolved_requirements(resolved_requirements, requirements, python_version, keep_tests=None, no_docker=False,
                                      build_directory='./build'):
    backend = _backend()
    warmup(backend, build_directory)  # the context comes up while the script below runs
    install_dir = build_directory if no_docker else '/tmp/export'
    pending = [r['line'] for r in requirements if resolved_requirements[r['requirement'].name] is None]
    pip_args = ''.join(' "%s"' % line for line in pending)
    if pending:
        print('Installing remaining packages via pip')

    # b200 backend: the rm lines (:256-259) and the strip line (:260) leave the script and happen on one
    # walk of the tree in the library; gnu/off keep the reference's rm lines where they are
    own_cleanup = backend == "b200"
    script_path = build_directory + '/build'
    with open(script_path, 'w') as f:
        f.write('\n'.join(_script_lines(install_dir, pip_args, keep_tests, cleanup_in_script=not own_cleanup)) + '\n')
    os.chmod(script_path, os.stat(script_path).st_mode | stat.S_IEXEC)
    with open(script_path) as f:
        print(f.read())

    if no_docker:
        print("Installing without docker...")
        return_code = subprocess.Popen([script_path]).wait()
        if return_code == 0:
            return_code = strip_build_tree(build_directory, backend, cleanup=own_cleanup, keep_tests=keep_tests)
        if return_code != 0:
            print("Error in building lambdipy build.")
            sys.exit(return_code)
    else:
        print("Installing in a docker container...")
        if backend == "b200":
            _context()  # no GPU / no library: fail before the container is pulled and started, not after
        from lambdipy.project_build import _run_command_in_docker  # the reference's container runner, unchanged
        try:
            _run_command_in_docker('%s/build' % install_dir, build_directory=build_directory, python_version=python_version)
            # the container wrote into the bind-mounted host directory (reference :179-184, uid :219);
            # like the reference, a failing strip does not abort a docker-mode build (exec rc unchecked, :227)
            if strip_build_tree(build_directory, backend, cleanup=own_cleanup, keep_tests=keep_tests) != 0:
                print("Error in building lambdipy build.")
        finally:
            if os.path.exists(script_path):
                os.remove(script_path)
        print('Finalizing the build')
        return

    print('Finalizing the build')
    os.remove(script_path)
