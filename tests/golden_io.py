"""Loader for the reference-generated golden vectors (tests/golden/make_golden.py) and for stored answers of the
reference's Python binding (`reference_answer`)."""
import json
import os

import numpy as np

from whatshap_b200._abi import FlatProblem, FlatSolution

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GROUPS = ("reference_cases", "fuzz", "synthetic")


def load(group):
    """Yields (label, FlatProblem, FlatSolution or None, error text)."""
    z = np.load(os.path.join(HERE, group + ".npz"))
    for i in range(int(z["n"])):
        g = lambda f, default=None: z[f"{i}.{f}"] if f"{i}.{f}" in z.files else default
        prob = FlatProblem(
            positions=g("positions"), read_off=g("read_off"), ent_col=g("ent_col"), ent_allele=g("ent_allele"),
            ent_phred=g("ent_phred"), read_ind=g("read_ind"), recombcost=g("recombcost"), n_ind=int(g("n_ind")),
            trios=g("trios", np.zeros(0, np.uint32)), distrust=bool(int(g("distrust"))), gt=g("gt"), gl=g("gl"),
        )
        error = str(g("error"))
        sol = None
        if not error:
            sol = FlatSolution(prob.n_cols, prob.n_reads, prob.n_ind)
            sol.cost = int(g("cost"))
            for f in ("path_index", "path_tv", "partition", "sr_allele", "sr_quality"):
                setattr(sol, f, g(f))
        yield str(g("label")), prob, sol, error


def check(solve, group):
    """Run `solve(problem) -> FlatSolution` on every case of a group; returns the case count."""
    n = 0
    for label, prob, want, error in load(group):
        try:
            got, gerr = solve(prob), ""
        except RuntimeError as e:
            got, gerr = None, str(e)
        assert gerr == error, (label, gerr, error)
        if want is not None:
            assert got.same_as(want), (label, got.diff(want))
        n += 1
    return n


_ANSWERS = {}


def reference_answer(module, key, live=None):
    """The reference's answer `key`, stored in tests/golden/<module>_answers.json.  Where the reference binding is
    available the caller passes its `live` answer (JSON-like): it must equal the stored copy, and WHMEC_RECORD_GOLDEN=1
    stores it instead.  Elsewhere the stored copy stands for the reference."""
    path = os.path.join(HERE, module + "_answers.json")
    if path not in _ANSWERS:
        _ANSWERS[path] = json.load(open(path)) if os.path.exists(path) else {}
    stored = _ANSWERS[path]
    if live is not None:
        live = json.loads(json.dumps(live))
        if os.environ.get("WHMEC_RECORD_GOLDEN") == "1":
            stored[key] = live
            with open(path, "w") as f:
                json.dump(stored, f, sort_keys=True, separators=(",", ":"))
        assert stored.get(key) == live, f"{key}: the reference's answer differs from the stored one in {path}"
    assert key in stored, f"{key}: no stored answer of the reference in {path}"
    return stored[key]
