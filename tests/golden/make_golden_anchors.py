"""
Generates tests/golden/hook_anchors.json: how often each anchor string of integration/apply_hook.py occurs in
the reference revision the other goldens were generated from (h2oai/datatable @ 3611640).  The hook only
inserts next to anchors that occur exactly once; tests/test_bench_contract.py checks the script's anchors
against this record, so that the check needs no copy of the reference.

    DATATABLE_REFERENCE_SRC=<reference source tree> python tests/golden/make_golden_anchors.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "integration"))
import apply_hook as ah  # noqa: E402

# anchor attribute of apply_hook -> file of the reference it is searched in
ANCHORS = {
    "INCLUDE_ANCHOR": "src/core/sort.cc", "OPTION_ANCHOR": "src/core/sort.cc",
    "REGISTER_ANCHOR": "src/core/sort.cc", "HOOK_ANCHOR": "src/core/sort.cc",
    "RED_INCLUDE_ANCHOR": "src/core/expr/fexpr_reduce_unary.cc",
    "RED_HELPER_ANCHOR": "src/core/expr/fexpr_reduce_unary.cc",
    "RED_LOOP_ANCHOR": "src/core/expr/fexpr_reduce_unary.cc",
    "EXT_ANCHOR": "ci/ext.py",
}


def count_anchors(ref):
    out = {}
    for name, rel in ANCHORS.items():
        with open(os.path.join(ref, rel)) as fh:
            text = fh.read()
        anchor = getattr(ah, name)
        out[name] = {"file": rel, "anchor": anchor, "count": text.count(anchor)}
    return out


if __name__ == "__main__":
    ref = os.environ.get("DATATABLE_REFERENCE_SRC", "")
    if not os.path.isdir(ref):
        sys.exit("set DATATABLE_REFERENCE_SRC to the reference's source tree")
    with open(os.path.join(HERE, "hook_anchors.json"), "w") as fh:
        json.dump({"reference": "h2oai/datatable @ 3611640 (1.2.0a)", "anchors": count_anchors(ref)}, fh, indent=1)
        fh.write("\n")
