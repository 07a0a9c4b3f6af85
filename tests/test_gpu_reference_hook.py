"""GPU: the REFERENCE itself, patched by integration/apply_hook.py so that its group() calls dtb_group
(option sort.b200), must give the stock CPU results -- the drop-in boundary exercised from the
reference's side.  Needs the patched build staged under oracle/_ref/patched (git-ignored; build() makes it from a
scratch copy of the reference's source tree where that is readable, see INTEGRATION.md B); skipped without it."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATCHED = os.path.join(ROOT, "oracle", "_ref", "patched")


def _run(script):
    if not os.path.exists(os.path.join(PATCHED, "datatable", "__init__.py")):
        pytest.skip("no patched reference build under oracle/_ref/patched: build() makes it only where the "
                    "reference's source tree is readable (DATATABLE_REFERENCE_SRC, or `reference` next to the repository)")
    lib = os.path.join(ROOT, "datatable_b200", "lib")                   # the patched extension links libdtb200.so
    env = dict(os.environ, PYTHONPATH=PATCHED,
               LD_LIBRARY_PATH=os.pathsep.join(p for p in (lib, os.environ.get("LD_LIBRARY_PATH")) if p))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "integration", script)],
                       env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


def test_patched_reference_matches_its_own_cpu_path():
    """option sort.b200: the reference's group() through dtb_group"""
    assert "GPU path == CPU path" in _run("check_hook.py")


def test_patched_reference_reducers_match_its_own_cpu_path():
    """option sort.b200_reducers: the reference's sum/mean/min/max/count through dtb_reduce, with its CPU
    group() and with sort.b200 on (the whole DT[:, reducers, by(k)] on the engine)"""
    out = _run("check_hook_reducers.py")
    assert out.count("engine == CPU for 12 reducers") == 2, out


def test_patched_reference_views_and_residency():
    """ArrayView_ColumnImpl::materialize through dtb_gather; the residency bracket around evaluate()"""
    out = _run("check_hook_views.py")
    assert "view columns on the engine == CPU path: ok" in out and "residency bracket): ok" in out, out
