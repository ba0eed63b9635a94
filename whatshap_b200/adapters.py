"""Running the CUDA solver on the reference's OWN objects (SURVEY.md §8(f) rank 1).

Inside a real `whatshap phase` run the ReadSet / Pedigree are the Cython objects of `whatshap.core`
(`readselect.pyx:244` reaches into `ReadSet.thisptr`, so they cannot be replaced); only the solver is
swapped by patching the name imported at `whatshap/cli/phase.py:34-42`.  This module provides that
swap-in class.  It touches the foreign objects only through their public Python API
(`whatshap/core.pyx:62-361,419-466`), so it works for this package's containers as well.

    import whatshap.core, whatshap.cli.phase, whatshap_b200.adapters as a
    whatshap.cli.phase.Pedigree = a.recording_pedigree(whatshap.core.Pedigree)
    whatshap.cli.phase.PedigreeDPTable = a.make_dp_table_class(whatshap.core)

The real `Pedigree` has no getter for its individuals or trio relationships; `recording_pedigree`
returns a subclass that remembers what it was given (cdef classes are subclassable from Python).
Without it the adapter falls back to parsing `str(pedigree)` (src/pedigree.cpp:91-123), which prints
genotype likelihoods with 6 significant digits — exact for the integer phred GLs WhatsHap produces
(`whatshap/vcf.py:269-285`), lossy for arbitrary doubles.
"""
from __future__ import annotations

import re
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _lib, multigpu
from ._abi import GT_OTHER, FlatProblem


def recording_pedigree(base):
    """Subclass of a `Pedigree` class that records individuals (name, numeric id, genotypes, GLs) and
    trio relationships as they are added."""

    class RecordingPedigree(base):
        def __init__(self, numeric_sample_ids):
            try:
                super().__init__(numeric_sample_ids)
            except TypeError:  # cdef class: __cinit__ already consumed the argument
                pass
            self._rec_ids = numeric_sample_ids
            self._rec_individuals = []  # (numeric id, genotypes, genotype likelihoods or None)
            self._rec_trios = []        # (father numeric id, mother numeric id, child numeric id)

        def add_individual(self, id, genotypes, genotype_likelihoods=None):
            genotypes = list(genotypes)
            gls = list(genotype_likelihoods) if genotype_likelihoods else None
            super().add_individual(id, genotypes, gls)
            self._rec_individuals.append((self._rec_ids[id], genotypes, gls))

        def add_relationship(self, father_id, mother_id, child_id):
            super().add_relationship(father_id, mother_id, child_id)
            self._rec_trios.append((self._rec_ids[father_id], self._rec_ids[mother_id], self._rec_ids[child_id]))

    RecordingPedigree.__name__ = "Recording" + base.__name__
    return RecordingPedigree


def _pedigree_from_recording(pedigree):
    ids = [numeric for numeric, _, _ in pedigree._rec_individuals]
    index = {numeric: i for i, numeric in enumerate(ids)}
    trios = [(index[f], index[m], index[c]) for f, m, c in pedigree._rec_trios]
    gts, gls = [], []
    for _, genotypes, likelihoods in pedigree._rec_individuals:
        gts.append([int(g.get_index()) if g.is_diploid_and_biallelic() else GT_OTHER for g in genotypes])
        if likelihoods is None:
            gls.append([None] * len(genotypes))
        else:
            gls.append([None if gl is None else [float(x) for x in list(gl)[:3]] for gl in likelihoods])
    return ids, trios, gts, gls


_GT_RE = re.compile(r"(\S+) \(GL:(None\)|PhredGenotypeLikelihoods\(([^\s)]*))")


def _pedigree_from_str(pedigree):
    text = str(pedigree)
    head = re.search(r"individuals \(index,id\):(.*)", text).group(1)
    ids = [int(tok.split(",")[1]) for tok in head.split()]
    trio_line = re.search(r"triples by index \(father,mother,child\):(.*)", text).group(1)
    trios = [tuple(int(x) for x in t.split(",")) for t in re.findall(r"\(([^)]*)\)", trio_line)]
    gts, gls = [], []
    blocks = re.split(r"individual index:\d+ / id:\d+:", text)[1:]
    for block in blocks:
        g_row, l_row = [], []
        for gt, none_or_gl, values in _GT_RE.findall(block):
            alleles = [] if gt == "." else [int(a) for a in gt.split("/")]
            ok = len(alleles) == 2 and all(a <= 1 for a in alleles)
            g_row.append(sum(alleles) if ok else GT_OTHER)
            l_row.append(None if none_or_gl.startswith("None") else [float(x) for x in values.split(",")][:3])
        gts.append(g_row)
        gls.append(l_row)
    return ids, trios, gts, gls


def _bridge_for(readset):
    """The compiled reference-side binding (integration/whatshap_bridge.pyx), if it is importable and
    `readset` is a genuine `whatshap.core.ReadSet`; else None."""
    if type(readset).__module__ != "whatshap.core":
        return None
    try:  # Cython re-checks every extension type of whatshap.core at import: a patched attribute there makes it refuse
        import whatshap_bridge
    except (ImportError, ValueError, TypeError):
        return None
    return whatshap_bridge


def _readset_to_csr(readset):
    """(read_off, ent_pos, ent_allele, ent_quality, sample_id, names or None) of any ReadSet-like object."""
    bridge = _bridge_for(readset)
    if bridge is not None:  # straight from the C++ objects, no Python object per entry
        off, pos, allele, quality, sample, _ = bridge.readset_to_csr(readset)
        return off.astype(np.int64), pos.astype(np.int64), allele.astype(np.int64), quality.astype(np.int64), sample.astype(np.int64), None
    off, pos, allele, quality, sample, names = [0], [], [], [], [], []
    for read in readset:
        for v in read:
            pos.append(v.position)
            allele.append(v.allele)
            quality.append(v.quality)
        off.append(len(pos))
        sample.append(read.sample_id)
        names.append(read.name)
    as_int = lambda xs: np.array(xs, np.int64)
    return as_int(off), as_int(pos), as_int(allele), as_int(quality), as_int(sample), names


def flatten_objects(readset, recombcost, pedigree, distrust_genotypes: bool = False, positions=None) -> Tuple[FlatProblem, List[int]]:
    """ReadSet / Pedigree objects of `whatshap.core` (or of this package) -> (`whmec_problem` arrays,
    numeric sample id of every pedigree index).  Errors of the reference's constructor path are raised with its
    texts (src/pedigreedptable.cpp:32-34, src/columniterator.cpp:29,32), the first offending read deciding."""
    if hasattr(pedigree, "_rec_individuals"):
        ids, trios, gts, gls = _pedigree_from_recording(pedigree)
    else:
        ids, trios, gts, gls = _pedigree_from_str(pedigree)
    pos_list = np.array(list(readset.get_positions()) if positions is None else [int(p) for p in positions], np.int64)
    n = len(pos_list)
    off, ent_pos, ent_allele, ent_quality, sample, names = _readset_to_csr(readset)
    n_reads = len(off) - 1
    name_of = lambda r: names[r] if names is not None else readset[int(r)].name
    lens = np.diff(off)
    id_arr = np.array(ids, np.int64)
    id_order = np.argsort(id_arr, kind="stable")
    slot = np.searchsorted(id_arr[id_order], sample)
    known = (slot < len(ids)) & (id_arr[id_order][np.minimum(slot, max(len(ids) - 1, 0))] == sample) if len(ids) else np.zeros(n_reads, bool)
    read_ind = id_order[np.minimum(slot, max(len(ids) - 1, 0))] if len(ids) else np.zeros(n_reads, np.int64)
    # per-read checks, in the order the reference meets them while walking the reads
    nonempty = lens > 0
    first = np.where(nonempty, ent_pos[np.minimum(off[:-1], max(len(ent_pos) - 1, 0))] if len(ent_pos) else 0, 0)
    last = np.where(nonempty, ent_pos[np.maximum(off[1:] - 1, 0)] if len(ent_pos) else 0, 0)
    prev_first = np.concatenate([[np.iinfo(np.int64).min], np.maximum.accumulate(first)[:-1]]) if n_reads else first
    inner_unsorted = np.zeros(n_reads, bool)
    if len(ent_pos) > 1:
        step_bad = np.diff(ent_pos) <= 0
        step_bad[off[1:-1][(off[1:-1] > 0) & (off[1:-1] < len(ent_pos))] - 1] = False  # steps across read boundaries
        read_of_step = np.repeat(np.arange(n_reads), lens)[:-1]
        inner_unsorted[np.unique(read_of_step[step_bad])] = True
    in_positions = lambda p: (np.searchsorted(pos_list, p) < n) & (pos_list[np.minimum(np.searchsorted(pos_list, p), max(n - 1, 0))] == p) if n else np.zeros(len(p), bool)
    ends_known = in_positions(first) & in_positions(last)
    bad_allele_entry = (ent_allele < 0) | (ent_allele > 2)
    ent_in_positions = in_positions(ent_pos)
    read_of_entry = np.repeat(np.arange(n_reads), lens)
    bad_allele = np.zeros(n_reads, bool)
    bad_allele[np.unique(read_of_entry[bad_allele_entry & ent_in_positions])] = True
    problems = [
        (~known, lambda r: "Individual with ID {} not present in pedigree.".format(int(sample[r]))),
        (~nonempty, lambda r: "No variants present"),
        (first < prev_first, lambda r: "ColumnIterator: reads in ReadSet are not sorted."),
        (inner_unsorted, lambda r: "ColumnIterator: encountered read with unsorted variants."),
        (~ends_known, lambda r: "read {!r}: first/last variant position is not among the given positions".format(name_of(r))),
        (bad_allele, lambda r: "read {!r}: allele {} is not 0, 1 or 2".format(
            name_of(r), int(ent_allele[off[r]:off[r + 1]][(bad_allele_entry & ent_in_positions)[off[r]:off[r + 1]]][0]))),
    ]
    any_bad = np.zeros(n_reads, bool)
    for mask, _ in problems:
        any_bad |= mask
    if any_bad.any():
        r = int(np.argmax(any_bad))
        for mask, message in problems:
            if mask[r]:
                raise RuntimeError(message(r))
    keep = ent_in_positions
    kept_per_read = np.add.reduceat(keep.astype(np.int64), off[:-1]) if n_reads else np.zeros(0, np.int64)
    read_off = np.concatenate([[0], np.cumsum(kept_per_read)]).astype(np.uint64)
    ent_col = np.searchsorted(pos_list, ent_pos[keep]).astype(np.uint32)
    n_ind = len(ids)
    rc = [int(x) for x in recombcost]
    if len(rc) < n:
        rc = rc + [rc[-1] if rc else 0] * (n - len(rc))
    gt = np.full((n_ind, n), GT_OTHER, np.uint8)
    gl = np.zeros((n_ind, n, 3), np.float64) if distrust_genotypes else None
    for i in range(n_ind):
        if n and len(gts[i]) < n:
            raise RuntimeError("pedigree holds genotypes for {} variants but the DP has {} columns".format(len(gts[i]), n))
        gt[i, :] = gts[i][:n]
        if distrust_genotypes:
            for k in range(n):
                if gls[i][k] is None:
                    raise RuntimeError("distrust_genotypes requires genotype likelihoods for every variant")
                gl[i, k, :] = gls[i][k]
    return FlatProblem(
        positions=pos_list.astype(np.uint32), read_off=read_off, ent_col=ent_col,
        ent_allele=ent_allele[keep].astype(np.uint8), ent_phred=ent_quality[keep].astype(np.uint32), read_ind=read_ind.astype(np.uint32),
        recombcost=np.array(rc[:n], np.uint32), n_ind=n_ind, trios=np.array([x for t in trios for x in t], np.uint32),
        distrust=bool(distrust_genotypes), gt=gt, gl=gl,
    ), ids


def _run_tables(problems, solver, tables_fn, device, devices):
    """Results of the `batch` classmethods of the swap-in classes (no per-table stats): `solver` on every problem, an exception
    in the table's place, or `tables_fn` (`multigpu.solve_tables` / `genotype_tables`) over all of them."""
    if not solver:
        return tables_fn(problems, device, devices), None
    results = []
    for p in problems:
        try:
            results.append(solver(p))
        except Exception as e:  # noqa: BLE001
            results.append(e)
    return results, None


def make_dp_table_class(core_module, solver=None):
    """A `PedigreeDPTable` look-alike (same constructor, same three methods, `whatshap/types.py:7-15`)
    that solves on the GPU and answers with `core_module`'s own Read / ReadSet objects.
    `solver(problem) -> FlatSolution` defaults to the CUDA path: device 0, or every GPU listed in WHMEC_DEVICES
    (`multigpu.solve_table`); tests may inject a CPU checker."""
    Read, ReadSet = core_module.Read, core_module.ReadSet

    class PedigreeDPTable:
        def __init__(self, readset, recombcost, pedigree, distrust_genotypes=False, positions=None):
            self.pedigree = pedigree
            self._problem, self._ids = flatten_objects(readset, recombcost, pedigree, distrust_genotypes, positions)
            solve = solver or (lambda p: multigpu.solve_table(p)[0])
            self._solution = solve(self._problem)

        @classmethod
        def batch(cls, tables, device=0, devices=None, return_exceptions=False):
            """Several tables in one call (`core.PedigreeDPTable.batch`): `tables` holds constructor argument tuples."""
            def build(obj, args):
                obj.pedigree = args[2]
                obj._problem, obj._ids = flatten_objects(args[0], args[1], args[2], args[3] if len(args) > 3 else False, args[4] if len(args) > 4 else None)

            return multigpu.batch_objects(cls, tables, build, lambda problems: _run_tables(problems, solver, multigpu.solve_tables, device, devices),
                                          "_solution", return_exceptions)

        def get_super_reads(self):
            prob, sol = self._problem, self._solution
            positions = prob.positions.tolist()
            results = []
            for k, numeric in enumerate(self._ids):
                rs = ReadSet()
                for h in range(2):
                    read = Read("superread_{}_{}".format(h, k), -1, -1, numeric)
                    for p, a, q in zip(positions, sol.sr_allele[k, h].tolist(), sol.sr_quality[k].tolist()):
                        read.add_variant(p, a, q)
                    rs.add(read)
                results.append(rs)
            return results, sol.path_tv.tolist()

        def get_optimal_cost(self):
            c = int(self._solution.cost)
            return c - (1 << 32) if c >= (1 << 31) else c

        def get_optimal_partitioning(self):
            return self._solution.partition.tolist()

    return PedigreeDPTable


def make_heuristic_class(core_module):
    """A `PedMecHeuristic` look-alike (constructor and methods of whatshap/core.pyx:674-734) for `core_module`'s own objects:
    `whatshap.cli.phase.PedMecHeuristic = make_heuristic_class(whatshap.core)` (name imported at cli/phase.py:41).  Runs the host
    solver `whmec_heuristic` (bit-identical to src/pedmecheuristic.cpp) and answers with `core_module`'s Read / ReadSet objects.
    The reference requires the reads' sample ids to be the zero-based indices of the pedigree's individuals."""
    Read, ReadSet = core_module.Read, core_module.ReadSet

    class PedMecHeuristic:
        def __init__(self, readset, recombcost, pedigree, row_limit=256, distrust_genotypes=False, positions=None, allow_mutations=True,
                     verbosity=0):
            self._setup(readset, recombcost, pedigree, distrust_genotypes, positions)
            self._solution = _lib.heuristic(self._problem, min(max(int(row_limit), 0), 65535), bool(allow_mutations))

        def _setup(self, readset, recombcost, pedigree, distrust_genotypes, positions):
            self.pedigree = pedigree
            # genotype likelihoods play no role in the heuristic: flatten with trusted genotypes, keep the flag for the solver
            self._problem, ids = flatten_objects(readset, recombcost, pedigree, False, positions)
            if list(ids) != list(range(len(ids))):
                raise RuntimeError("PedMecHeuristic: sample ids must be the zero-based indices of the pedigree's individuals")
            self._problem.distrust = bool(distrust_genotypes)
            self._sample_ids = sorted(set(self._problem.read_ind.tolist()) | set(self._problem.trios.tolist()))

        @classmethod
        def batch(cls, tables, device=0, devices=None, return_exceptions=False):
            """Several tables in one call (`core.PedMecHeuristic.batch`): `tables` holds constructor argument tuples."""
            def setup(obj, args):
                obj._setup(args[0], args[1], args[2], args[4] if len(args) > 4 else False, args[5] if len(args) > 5 else None)

            return multigpu.batch_heuristic_objects(cls, tables, setup, device, devices, return_exceptions)

        def get_super_reads(self):
            prob, sol = self._problem, self._solution
            positions = prob.positions.tolist()
            results = []
            for k, sid in enumerate(self._sample_ids):
                rs = ReadSet()
                for h in range(2):
                    read = Read("superread_{}".format(h), -1, -1, sid)
                    for p, a in zip(positions, sol.haplotypes[k, h].tolist()):
                        read.add_variant(p, a, 30)
                    rs.add(read)
                results.append(rs)
            return results, sol.transmission.tolist()

        def get_optimal_cost(self):
            return float(self._solution.score)

        def get_optimal_partitioning(self):
            return [0 if x else 1 for x in self._solution.partition.tolist()]

        def get_mutations(self):
            sol, out = self._solution, []
            for k in range(sol.n_samples):
                cols, haps = np.nonzero(sol.mutated[k].T)
                out.append([(int(h), int(c)) for c, h in zip(cols, haps)])
            return out

    return PedMecHeuristic


def make_genotype_table_class(core_module, solver=None):
    """A `GenotypeDPTable` look-alike (constructor and `get_genotype_likelihoods` of whatshap/core.pyx:581-600) that
    runs the forward-backward DP on the GPU from `core_module`'s own objects and answers with its
    `PhredGenotypeLikelihoods`.  The pedigree should be a `recording_pedigree` (exact genotype priors; the `str()`
    fallback keeps 6 significant digits).  `solver(problem) -> ndarray [n_ind, n_cols, 3]` defaults to the CUDA path: device
    0, or every GPU listed in WHMEC_DEVICES (`multigpu.genotype_table`)."""
    Likelihoods = core_module.PhredGenotypeLikelihoods

    class GenotypeDPTable:
        def __init__(self, numeric_sample_ids, readset, recombcost, pedigree, positions=None):
            self.pedigree = pedigree
            self.numeric_sample_ids = numeric_sample_ids
            # the priors travel where distrusted genotypes carry their likelihoods
            self._problem, self._ids = flatten_objects(readset, recombcost, pedigree, True, positions)
            run = solver or (lambda p: multigpu.genotype_table(p)[0])
            self._likelihoods = run(self._problem)

        @classmethod
        def batch(cls, tables, device=0, devices=None, return_exceptions=False):
            """Several tables in one call (`core.GenotypeDPTable.batch`): `tables` holds constructor argument tuples."""
            def build(obj, args):
                obj.pedigree = args[3]
                obj.numeric_sample_ids = args[0]
                obj._problem, obj._ids = flatten_objects(args[1], args[2], args[3], True, args[4] if len(args) > 4 else None)

            return multigpu.batch_objects(cls, tables, build, lambda problems: _run_tables(problems, solver, multigpu.genotype_tables, device, devices),
                                          "_likelihoods", return_exceptions)

        def get_genotype_likelihoods(self, sample_id, pos):
            index = self._ids.index(self.numeric_sample_ids[sample_id])
            if not 0 <= pos < self._problem.n_cols:
                raise IndexError("position index out of range")
            return Likelihoods(self._likelihoods[index, pos].tolist())

    return GenotypeDPTable


def make_compute_genotypes(core_module):
    """`compute_genotypes(readset, positions=None)` (whatshap/core.pyx:602-617) for `core_module`'s own ReadSet objects:
    per-variant genotype priors through `whmec_compute_genotypes` (host; identical doubles), answered with
    `core_module.Genotype` objects and likelihood tuples."""
    Genotype = core_module.Genotype

    class _Het:  # any genotype will do: the prior genotyper looks at the reads only
        @staticmethod
        def is_diploid_and_biallelic():
            return True

        @staticmethod
        def get_index():
            return 1

    def compute_genotypes(readset, positions=None):
        n = len(readset.get_positions()) if positions is None else len(positions)
        samples = sorted({int(read.sample_id) for read in readset}) or [0]
        stub = type("ReadsOnly", (), {})()
        stub._rec_individuals = [(sid, [_Het] * n, None) for sid in samples]
        stub._rec_trios = []
        prob, _ = flatten_objects(readset, [0] * n, stub, False, positions)
        gl, gt = _lib.compute_genotypes(prob)
        alleles = ([0, 0], [0, 1], [1, 1])
        return [Genotype(alleles[g]) if g >= 0 else Genotype([]) for g in gt.tolist()], [tuple(row) for row in gl.tolist()]

    return compute_genotypes


def make_prepare_haplotag_information(haplotag_module):
    """`prepare_haplotag_information` (whatshap_b200.haplotag) with its keys built from `haplotag_module`'s own
    ReadAlignmentRepresentation and PrimaryInfo, so that assigning it in place of the reference's function lets an unchanged
    `run_haplotag` look the reads up (a dataclass compares equal only to instances of its own class):

        import whatshap.cli.haplotag as h, whatshap_b200.adapters as a
        h.prepare_haplotag_information = a.make_prepare_haplotag_information(h)
    """
    from . import haplotag

    repr_cls, info_cls = haplotag_module.ReadAlignmentRepresentation, haplotag_module.PrimaryInfo

    def prepare_haplotag_information(variant_table, shared_samples, phased_input_reader, regions, ignore_linked_read, linked_read_cutoff,
                                     ploidy, supplementary_strategy=None, *, device=0, stats=None, library=None):
        return haplotag._prepare(repr_cls, info_cls, variant_table, shared_samples, phased_input_reader, regions, ignore_linked_read,
                                 linked_read_cutoff, ploidy, device, stats, library)

    return prepare_haplotag_information
