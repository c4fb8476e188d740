"""Pins the statement-level metric to the reference's OWN code — by running it.

DDFA/sastvd/helpers/evaluate.py:262-322 (eval_statements, eval_statements_inter, eval_statements_list) is IVDetect's top-k
statement accuracy.  The module imports the reference's dataset / tokeniser / Joern helpers at the top, which pull in the rest of
its data pipeline; none of them is used by these three functions.  This script installs empty stand-ins for those helper modules
(as make_reference_ctrlflow_golden.py does for the packages the model code imports), loads evaluate.py itself and runs
eval_statements_list on seeded cases:

    ties (scores on a coarse grid), functions of fewer than 10 statements, single-statement functions, a clean function whose
    largest probability is exactly 0.5 and one just above it, all-vulnerable functions, functions of up to thousands of
    statements, and both vo=True and vo=False.

Run with a checkout of the reference project:   python tests/golden/make_reference_statement_golden.py <reference root>
Writes tests/golden/reference_statement_golden.pt, read by tests/test_statements_cpu.py and tests/test_statements_gpu.py: per
case the fp32 scores and _VULN labels in node order, the statement count of every function, and the reference's outputs (None
where the reference divides by zero).
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def install_stand_ins():
    """The reference helper modules evaluate.py imports at the top but eval_statements* never calls."""
    names = ["sastvd", "sastvd.helpers", "sastvd.helpers.datasets", "sastvd.helpers.tokenise", "sastvd.helpers.joern"]
    mods = {n: types.ModuleType(n) for n in names}
    mods["sastvd"].helpers = mods["sastvd.helpers"]
    for n in names[2:]:
        setattr(mods["sastvd.helpers"], n.rsplit(".", 1)[1], mods[n])
    sys.modules.update(mods)


def load_evaluate(reference_root):
    install_stand_ins()
    path = os.path.join(reference_root, "DDFA", "sastvd", "helpers", "evaluate.py")
    spec = importlib.util.spec_from_file_location("reference_evaluate", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def make_case(rng, sizes, vuln_rate, grid, all_vuln=False, clean_specials=False):
    """Functions of the given statement counts; probabilities on a grid of `grid` steps (ties) or continuous (grid=0)."""
    scores, labels = [], []
    for i, n in enumerate(sizes):
        if grid:
            p = rng.integers(0, grid + 1, size=n).astype(np.float64) / grid
        else:
            p = rng.random(n)
        p = p.astype(np.float32)
        if all_vuln:
            y = np.ones(n, dtype=np.int32)
        elif rng.random() < vuln_rate:
            y = (rng.random(n) < 0.3).astype(np.int32)
            if y.sum() == 0:
                y[rng.integers(0, n)] = 1
        else:
            y = np.zeros(n, dtype=np.int32)
        scores.append(p)
        labels.append(y)
    if clean_specials:
        # non-vulnerable: the largest probability exactly 0.5 (clean: the comparison is strict), and one ulp above it (not clean)
        for v in (np.float32(0.5), np.nextafter(np.float32(0.5), np.float32(1.0))):
            p = np.full(7, 0.25, dtype=np.float32)
            p[3] = v
            scores.append(p)
            labels.append(np.zeros(7, dtype=np.int32))
    return scores, labels


def main(reference_root):
    ev = load_evaluate(reference_root)
    rng = np.random.default_rng(20261017)
    specs = [
        ("ties_small", dict(sizes=list(rng.integers(1, 15, size=60)) + [1, 1, 1, 2, 9, 10, 11], vuln_rate=0.5, grid=8, clean_specials=True)),
        ("continuous", dict(sizes=list(rng.integers(1, 40, size=50)), vuln_rate=0.4, grid=0, clean_specials=True)),
        ("single_statement", dict(sizes=[1] * 30, vuln_rate=0.5, grid=4)),
        ("all_vulnerable", dict(sizes=[1, 3, 12, 40], vuln_rate=1.0, grid=4, all_vuln=True)),
        ("large_ties", dict(sizes=[3000, 1500, 257, 129, 5, 640], vuln_rate=0.7, grid=64, clean_specials=True)),
        ("no_vulnerable", dict(sizes=[4, 6, 20], vuln_rate=0.0, grid=16, clean_specials=True)),
    ]
    cases = []
    for name, spec in specs:
        scores, labels = make_case(rng, **spec)
        items = [[[[1.0 - float(q), float(q)] for q in p], [int(v) for v in y]] for p, y in zip(scores, labels)]
        out = {}
        for vo in (True, False):
            try:
                r = ev.eval_statements_list(items, thresh=0.5, vo=vo)
                out[vo] = {int(k): float(v) for k, v in r.items()}
            except ZeroDivisionError:
                out[vo] = None
        cases.append({"name": name, "scores": torch.from_numpy(np.concatenate(scores)),
                      "vuln": torch.from_numpy(np.concatenate(labels)),
                      "batch_num_nodes": torch.tensor([len(p) for p in scores], dtype=torch.int64),
                      "vo": out[True], "all": out[False]})
    path = os.path.join(ROOT, "tests", "golden", "reference_statement_golden.pt")
    torch.save({"cases": cases, "note": "outputs of the reference's own evaluate.py eval_statements_list (thresh=0.5)"}, path)
    print("wrote", path, {c["name"]: int(c["batch_num_nodes"].numel()) for c in cases})


if __name__ == "__main__":
    main(sys.argv[1])
