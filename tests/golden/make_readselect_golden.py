"""Generates tests/golden/readselect.npz with the UNMODIFIED reference: `whatshap.readselect.readselection`
and `whatshap.priorityqueue.PriorityQueue`, built out of tree by oracle/build_pyref.py from the
WhatsHap tree at $WHATSHAP_REF (a Python reference cannot travel to a machine without it, its outputs can).
    python tests/golden/make_readselect_golden.py

Contents
  rs.<j>.*    read sets as CSR (read_off, ent_var -> positions, ent_quality, source_id)
  sel.<i>.*   read set number, the arguments (max_cov, bridging, preferred source ids) and the sorted indices
              the reference selects.  Which read wins a tie
              depends on CPython's set iteration order: valid for the CPython 3.12 set implementation.
  pq.<i>.*    operation traces on the reference's priority queue (op, item, score) and what every pop /
              get_score_by_item returned.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import build_pyref  # noqa: E402

PYREF = build_pyref.build()
assert PYREF, "the reference tree is needed to generate golden vectors"
sys.path.insert(0, PYREF)

import whatshap.core as wc  # noqa: E402
from whatshap.priorityqueue import PriorityQueue  # noqa: E402
from whatshap.readselect import readselection  # noqa: E402


def random_reads(rng, n_var, n_reads, mean_len, gap, n_sources, max_quality):
    """Reads over `n_var` variant positions: geometric lengths, interior gaps, in ReadSet (start) order."""
    positions = np.sort(rng.choice(np.arange(1, 20 * n_var), n_var, replace=False)).astype(int)
    reads = []
    for _ in range(n_reads):
        start = int(rng.integers(0, n_var - 1))
        idx = np.arange(start, min(n_var, start + 2 + int(rng.geometric(1.0 / mean_len))))
        if len(idx) > 2 and gap > 0:
            keep = rng.random(len(idx)) >= gap
            keep[0] = keep[-1] = True
            idx = idx[keep]
        if len(idx) < 2:
            continue
        reads.append((int(rng.integers(0, n_sources)), positions[idx], rng.integers(1, max_quality, len(idx)), idx))
    reads.sort(key=lambda r: int(r[1][0]))
    return reads, positions


def to_reference_readset(reads):
    rs = wc.ReadSet()
    for i, (source, pos, qual, _) in enumerate(reads):
        read = wc.Read("r%d" % i, 50, source, 0)
        for p, q in zip(pos.tolist(), qual.tolist()):
            read.add_variant(p, q & 1, q)
        rs.add(read)
    return rs


def selection_cases():
    rng = np.random.default_rng(20250923)
    out, i, j = {}, 0, 0
    for it in range(90):
        n_var, n_reads = int(rng.integers(5, 160)), int(rng.integers(2, 300))
        reads, positions = random_reads(rng, n_var, n_reads, float(rng.choice([2, 5, 15])), float(rng.choice([0, 0.2, 0.5])),
                             int(rng.integers(1, 4)), int(rng.choice([3, 60])))
        if not reads:
            continue
        rs = to_reference_readset(reads)
        out[f"rs.{j}.read_off"] = np.cumsum([0] + [len(r[1]) for r in reads]).astype(np.uint32)
        out[f"rs.{j}.positions"] = positions.astype(np.int32)  # ent_pos = positions[ent_var]
        out[f"rs.{j}.ent_var"] = np.concatenate([r[3] for r in reads]).astype(np.uint8)
        out[f"rs.{j}.ent_quality"] = np.concatenate([r[2] for r in reads]).astype(np.uint8)
        out[f"rs.{j}.source_id"] = np.array([r[0] for r in reads], np.uint8)
        for max_cov, bridging, preferred in ((1, False, None), (2, True, None), (5, True, {1}), (15, True, {0, 2}), (3, False, {2})):
            chosen = readselection(rs, max_cov, preferred, bridging)
            out[f"sel.{i}.args"] = np.array([j, max_cov, int(bridging)], np.int32)
            out[f"sel.{i}.preferred"] = np.array(sorted(preferred) if preferred is not None else [-1], np.int32)
            out[f"sel.{i}.selected"] = np.array(sorted(chosen), np.int32)
            i += 1
        j += 1
    out["sel.n"] = np.array(i)
    return out


def queue_traces():
    rng = np.random.default_rng(7)
    out = {}
    for t in range(40):
        width = int(rng.choice([1, 3]))
        top = int(rng.choice([3, 50]))  # small range: many ties
        pq, queued, ops, answers = PriorityQueue(), [], [], []
        score = lambda: [int(x) for x in rng.integers(0, top, width)] + [0] * (3 - width)
        for _ in range(int(rng.integers(20, 200))):
            kind = int(rng.integers(0, 4))
            if kind == 0 or not queued:
                item = int(rng.integers(0, 10_000))
                if item in queued:
                    continue
                s = score()
                pq.push(tuple(s[:width]) if width > 1 else s[0], item)
                queued.append(item)
                ops.append([0, item] + s)
            elif kind == 1:
                s, item = pq.pop()
                queued.remove(item)
                ops.append([1, 0, 0, 0, 0])
                answers.append([item] + (list(s) if width > 1 else [s, 0, 0]))
            elif kind == 2:
                item, s = queued[int(rng.integers(0, len(queued)))], score()
                pq.change_score(item, tuple(s[:width]) if width > 1 else s[0])
                ops.append([2, item] + s)
            else:
                item = queued[int(rng.integers(0, len(queued)))]
                s = pq.get_score_by_item(item)
                ops.append([3, item, 0, 0, 0])
                answers.append([item] + (list(s) if width > 1 else [s, 0, 0]))
        while len(pq):
            s, item = pq.pop()
            ops.append([1, 0, 0, 0, 0])
            answers.append([item] + (list(s) if width > 1 else [s, 0, 0]))
        out[f"pq.{t}.width"] = np.array(width)
        out[f"pq.{t}.ops"] = np.array(ops, np.int32).reshape(-1, 5)
        out[f"pq.{t}.answers"] = np.array(answers, np.int32).reshape(-1, 4)
    out["pq.n"] = np.array(40)
    return out


def ragged(data):
    """Few big arrays instead of thousands of zip members: fields `<group>.<i>.<name>` of equal dtype are
    concatenated to `<group>.<name>` with row offsets `<group>.<name>.off` (tests/test_readselect.py: unragged)."""
    out, groups = {}, {}
    for key, value in data.items():
        parts = key.split(".")
        if len(parts) != 3:
            out[key] = value
            continue
        groups.setdefault((parts[0], parts[2]), {})[int(parts[1])] = np.atleast_1d(value)
    for (group, name), rows in groups.items():
        ordered = [rows[i] for i in range(len(rows))]
        out[f"{group}.{name}"] = np.concatenate([r.reshape(-1) for r in ordered])
        out[f"{group}.{name}.off"] = np.cumsum([0] + [r.size for r in ordered]).astype(np.uint32)
    return out


if __name__ == "__main__":
    data = selection_cases()
    data.update(queue_traces())
    data = ragged(data)
    path = os.path.join(HERE, "readselect.npz")
    np.savez_compressed(path, **data)
    print(path, os.path.getsize(path) // 1024, "KiB;", int(data["sel.n"]), "selections,", int(data["pq.n"]), "queue traces")
