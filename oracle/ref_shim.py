"""Import shims that let the UNMODIFIED reference package (goktug97/estorch, installed by
``install_reference()`` during ``__graft_entry__.build()`` into ``oracle/_ref`` -- git-ignored, never
copied into this repo's sources) run in a single process: a one-rank ``mpi4py`` stand-in (the reference imports it at
estorch.py:10; with ``n_proc=1`` no MPI call is made, :207-209/:228-233 loop over zero workers) and
``np.int = int`` (estorch.py:453 uses the alias numpy removed).  TEST / BENCH INFRASTRUCTURE ONLY:
used by tests/golden/make_golden.py-style scripts and by ``bench.py --impl reference``."""
import os
import shutil
import subprocess
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
REF_EXAMPLES = os.path.join(REF_DIR, "examples")
# where the reference's source tree is checked out, when it is (override: ESTORCH_REFERENCE_SRC)
REF_SRC = os.environ.get("ESTORCH_REFERENCE_SRC", "/root/reference")


def install_reference() -> bool:
    """pip install --no-index --no-deps --target oracle/_ref <copy of the reference source tree>, plus a
    copy of its examples/ (read by tests/test_reference_examples_cpu.py).  The source tree may be
    read-only and setuptools writes build/ next to setup.py, hence the temporary copy.  Without the
    source tree nothing is installed and the reference arms fall back to oracle/reference_port.py."""
    if os.path.isdir(os.path.join(REF_DIR, "estorch")) or not os.path.isdir(REF_SRC):
        return os.path.isdir(os.path.join(REF_DIR, "estorch"))
    tmp = tempfile.mkdtemp(prefix="estorch_ref_")
    try:
        shutil.copytree(REF_SRC, os.path.join(tmp, "src"))
        r = subprocess.run([sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps",
                            "--target", REF_DIR, os.path.join(tmp, "src")], capture_output=True, text=True)
        if r.returncode != 0:
            print("reference install failed (bench.py --impl reference falls back to the CPU port):\n" + r.stderr[-800:])
            return False
        if os.path.isdir(os.path.join(REF_SRC, "examples")):
            shutil.copytree(os.path.join(REF_SRC, "examples"), REF_EXAMPLES, dirs_exist_ok=True)
        return True
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def install_shims():
    if "mpi4py" not in sys.modules:
        m = types.ModuleType("mpi4py")
        MPI = types.ModuleType("mpi4py.MPI")

        class _Comm:
            def Get_rank(self):
                return 0

            def Get_size(self):
                return 1

            def send(self, *a, **k):
                pass

            def bcast(self, x, root=0):
                return x

        class Status:
            def Get_tag(self):
                return 0

        MPI.COMM_WORLD, MPI.Status, m.MPI = _Comm(), Status, MPI
        sys.modules["mpi4py"], sys.modules["mpi4py.MPI"] = m, MPI
    if not hasattr(np, "int"):
        np.int = int


def import_reference():
    """The reference's ``estorch`` module from oracle/_ref, or None when it is not installed."""
    if not os.path.isdir(os.path.join(REF_DIR, "estorch")):
        return None
    install_shims()
    if REF_DIR not in sys.path:
        sys.path.insert(0, REF_DIR)
    try:
        import estorch  # noqa: F401  (the reference)
    except Exception:
        return None
    return sys.modules["estorch"]
