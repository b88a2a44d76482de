"""Every public top-level name of the reference exists in this package (or is a documented absence).  The reference's names
are stored in ``tests/golden/reference_public_names.json`` (written by ``tools/api_diff.py --dump`` from a reference checkout)."""
import importlib.util
import json
import os


def test_no_unexplained_missing_public_names():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("api_diff", os.path.join(root, "tools", "api_diff.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    with open(os.path.join(root, "tests", "golden", "reference_public_names.json")) as f:
        ref = json.load(f)
    assert sum(len(v) for v in ref.values()) > 500, "stored reference names look truncated"
    missing = mod.diff_names(ref, os.path.join(root, "neuronx_distributed_b200"))
    assert not missing, missing
