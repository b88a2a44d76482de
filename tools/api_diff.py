#!/usr/bin/env python
"""Public-surface diff against the reference checkout: every top-level, non-underscore ``def`` / ``class`` of every module under
``<reference>/src/neuronx_distributed`` must exist *somewhere* in ``neuronx_distributed_b200`` (module placement is checked
separately by ``tests/test_public_api.py``), except the names listed in ``ABSENT`` with the reason they have no CUDA
counterpart.  The reference's names are stored in ``tests/golden/reference_public_names.json`` so the check runs without the
reference checkout.

    python tools/api_diff.py --reference <checkout>                 # exit code 1 if an unexplained name is missing
    python tools/api_diff.py --reference <checkout> --dump FILE     # (re)write the stored reference names
    python tools/api_diff.py --names tests/golden/reference_public_names.json
"""
from __future__ import annotations

import argparse
import ast
import json
import os
import sys
from typing import Dict, List, Set

ABSENT: Dict[str, str] = {
    # modules/moe/nki_import.py, modules/moe/blockwise.py — loading NKI kernel packages at import time
    "NKIImport": "NKI kernel-package import machinery (kernels here are one in-tree CUDA extension)",
    "import_nki": "same",
    "import_nki_beta2": "same",
    "initialize_nki_components": "same",
    "initialize_training_kernels": "same",
}


def top_level_names(path: str) -> List[str]:
    try:
        tree = ast.parse(open(path).read())
    except SyntaxError:
        return []
    return [n.name for n in tree.body if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and not n.name.startswith("_")]


def our_names(pkg_root: str) -> Set[str]:
    names: Set[str] = set()
    for dp, _, files in os.walk(pkg_root):
        for f in files:
            if not f.endswith(".py"):
                continue
            try:
                tree = ast.parse(open(os.path.join(dp, f)).read())
            except SyntaxError:
                continue
            for n in tree.body:
                if isinstance(n, (ast.FunctionDef, ast.ClassDef)):
                    names.add(n.name)
                elif isinstance(n, ast.Assign):
                    names.update(t.id for t in n.targets if isinstance(t, ast.Name))
                elif isinstance(n, ast.ImportFrom):
                    names.update(a.asname or a.name for a in n.names)
                elif isinstance(n, (ast.If, ast.Try)):            # conditional definitions (optional dependencies)
                    for sub in ast.walk(n):
                        if isinstance(sub, (ast.FunctionDef, ast.ClassDef)):
                            names.add(sub.name)
                        elif isinstance(sub, ast.Assign):
                            names.update(t.id for t in sub.targets if isinstance(t, ast.Name))
    return names


def reference_names(reference: str) -> Dict[str, List[str]]:
    """Public top-level names of every module of a reference checkout, by path relative to its package root."""
    ref_root = os.path.join(reference, "src", "neuronx_distributed")
    out: Dict[str, List[str]] = {}
    for dp, _, files in sorted(os.walk(ref_root)):
        for f in sorted(files):
            if f.endswith(".py"):
                names = top_level_names(os.path.join(dp, f))
                if names:
                    out[os.path.relpath(os.path.join(dp, f), ref_root)] = names
    return out


def diff_names(ref: Dict[str, List[str]], pkg_root: str) -> Dict[str, List[str]]:
    have = our_names(pkg_root)
    missing: Dict[str, List[str]] = {}
    for rel, names in sorted(ref.items()):
        m = [n for n in names if n not in have and n not in ABSENT]
        if m:
            missing[rel] = m
    return missing


def diff(reference: str, pkg_root: str) -> Dict[str, List[str]]:
    return diff_names(reference_names(reference), pkg_root)


def main() -> int:
    ap = argparse.ArgumentParser()
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--reference", help="reference checkout")
    src.add_argument("--names", help="stored reference names (JSON)")
    ap.add_argument("--dump", help="write the reference's names to this JSON file")
    a = ap.parse_args()
    here = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "neuronx_distributed_b200")
    ref = reference_names(a.reference) if a.reference else json.load(open(a.names))
    if a.dump:
        with open(a.dump, "w") as f:
            json.dump(ref, f, indent=1, sort_keys=True)
            f.write("\n")
    missing = diff_names(ref, here)
    for mod, names in missing.items():
        print(f"{mod}: {names}")
    print(f"{sum(len(v) for v in missing.values())} unexplained missing names; {len(ABSENT)} documented absences")
    return 1 if missing else 0


if __name__ == "__main__":
    sys.exit(main())
