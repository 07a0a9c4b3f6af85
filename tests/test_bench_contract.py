"""CPU: the parts of bench.py and integration/ that run without a GPU keep their contracts."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` (the CPU leg: oracle port on all host threads) prints ONE JSON line with
    the keys the driver reads."""
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                        "--warmup", "1", "--cpu-rows", "300000"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1, r.stdout
    j = json.loads(lines[0])
    assert j["impl"] == "reference" and j["metric"].startswith("rows/sec groupby-sum")
    assert j["unit"] == "rows/s" and j["higher_is_better"] is True and j["value"] > 0
    cb = j["cpu_baseline"]
    assert cb["kind"] in ("port", "reference") and cb["cores"] >= 1 and cb["value"] == j["value"] and cb["sample"]
    assert j["e2e"]["value"] == j["value"] and j["e2e"]["h2d_bytes_per_step"] == 0 and j["e2e"]["d2h_bytes_per_step"] == 0
    assert j["steps"] == 1 and "workload" in j["config"]


def test_hook_script_anchors_match_the_reference(tmp_path):
    """integration/apply_hook.py inserts next to short anchor strings: each must occur exactly once in the
    reference revision the goldens were generated from (tests/golden/hook_anchors.json, recounted in the
    reference tree itself where DATATABLE_REFERENCE_SRC names one), and the script must refuse to touch
    the configured reference source tree or anything inside it."""
    sys.path.insert(0, os.path.join(ROOT, "integration"))
    try:
        import apply_hook as ah
    finally:
        sys.path.pop(0)
    src = tmp_path / "reference"
    (src / "src").mkdir(parents=True)
    for tree in (src, src / "src"):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "integration", "apply_hook.py"), str(tree)],
                           env=dict(os.environ, DATATABLE_REFERENCE_SRC=str(src)), capture_output=True, text=True)
        assert r.returncode != 0 and "refusing" in (r.stdout + r.stderr)
    with open(os.path.join(ROOT, "tests", "golden", "hook_anchors.json")) as fh:
        recorded = json.load(fh)["anchors"]
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        import make_golden_anchors as mga
    finally:
        sys.path.pop(0)
    assert set(recorded) == set(mga.ANCHORS)
    for name, rec in recorded.items():
        assert rec["anchor"] == getattr(ah, name), f"{name} changed since the anchors were counted in the reference"
        assert rec["count"] == 1, name
    ref = os.environ.get("DATATABLE_REFERENCE_SRC", "")
    if os.path.isdir(ref):
        assert all(rec["count"] == 1 for rec in mga.count_anchors(ref).values())
