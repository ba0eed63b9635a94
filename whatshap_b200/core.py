"""Host-side mirror of the reference's operator surface for the weighted-MEC / PedMEC DP.

Same names, argument meaning and error behaviour as the Cython classes of the reference
(`whatshap/core.pyx`): `NumericSampleIds` (:24-59), `Read` (:62-273), `ReadSet` (:275-361),
`PedigreeDPTable` (:364-416), `Pedigree` (:419-466), `PhredGenotypeLikelihoods` (:469-504),
`Genotype` (:511-570).  The containers are plain Python (they only hold data); the dynamic
program itself — everything `PedigreeDPTable.__cinit__` triggers in the reference — runs in
CUDA behind the C ABI of `include/whmec.h` (`whatshap_b200/_lib.py`).  There is no CPU
fallback: constructing a `PedigreeDPTable` without the CUDA library or a GPU raises.
"""
from __future__ import annotations

import copy
from array import array
from itertools import chain
from math import comb
from typing import Dict, Iterable, Iterator, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib, multigpu
from ._abi import GT_OTHER, FlatProblem, FlatSolution
from .variant import Variant

MAX_GENOTYPE_PLOIDY = 15   # src/genotype.h:58
MAX_GENOTYPE_ALLELES = 16  # src/genotype.h:53


class NumericSampleIds:
    """Mapping of sample names to numeric ids; unknown names are assigned the next id unless
    frozen (core.pyx:24-59)."""

    def __init__(self):
        self.mapping: Dict[str, int] = {}
        self.frozen = False

    def __getitem__(self, sample):
        if not self.frozen and sample not in self.mapping:
            self.mapping[sample] = len(self.mapping)
        return self.mapping[sample]

    def __len__(self):
        return len(self.mapping)

    def __str__(self):
        return str(self.mapping)

    def freeze(self):
        self.frozen = True

    def inverse_mapping(self):
        return {numeric_id: name for name, numeric_id in self.mapping.items()}

    def __getstate__(self):
        return (self.mapping, self.frozen)

    def __setstate__(self, state):
        self.mapping, self.frozen = state


def _typed(values) -> array:
    """array('q') from a numpy array or a sequence of ints."""
    out = array("q")
    if isinstance(values, np.ndarray):
        out.frombytes(np.ascontiguousarray(values, np.int64).tobytes())
    else:
        out.extend(values)
    return out


def _distinct_sorted(values: np.ndarray) -> np.ndarray:
    """Sorted distinct values of an int64 array (np.sort + neighbour comparison: several times faster than np.unique)."""
    if values.size == 0:
        return values
    s = np.sort(values)
    keep = np.empty(s.size, np.bool_)
    keep[0] = True
    np.not_equal(s[1:], s[:-1], out=keep[1:])
    return s[keep]


class Read:
    """A read: metadata plus (position, allele, quality) variants (core.pyx:62-273, src/read.cpp)."""

    __slots__ = (
        "_name", "_mapqs", "_source_id", "_sample_id", "_reference_start", "_reference_end", "_BX_tag", "_HP_tag",
        "_PS_tag", "_chromosome", "_sub_alignment_id", "_is_supplementary", "_is_reverse", "_pos", "_allele", "_quality",
        "_owner",
    )

    def __init__(self, name: Optional[str] = None, mapq: int = 0, source_id: int = 0, sample_id: int = 0,
                 reference_start: int = -1, BX_tag: Optional[str] = None, HP_tag: int = -1, PS_tag: int = -1,
                 chromosome: Optional[str] = None, sub_alignment_id: Optional[str] = None,
                 is_supplementary: bool = False, reference_end: int = -1, is_reverse: bool = False):
        self._name = name
        self._mapqs = [int(mapq)]
        self._source_id = int(source_id)
        self._sample_id = int(sample_id)
        self._reference_start = int(reference_start)
        self._reference_end = int(reference_end)
        self._BX_tag = BX_tag or ""
        self._HP_tag = int(HP_tag)
        self._PS_tag = int(PS_tag)
        self._chromosome = chromosome or ""
        self._sub_alignment_id = sub_alignment_id or ""
        self._is_supplementary = bool(is_supplementary)
        self._is_reverse = bool(is_reverse)
        # variants as three typed arrays (array('q')): appended to like lists, read by `_flatten_reads` through the buffer
        # protocol without a Python object per entry
        self._pos = array("q")
        self._allele = array("q")
        self._quality = array("q")
        self._owner = None  # the ReadSet this object is stored in (its columnar copy of the variants is dropped when the read changes)

    def _touch(self):
        if self._owner is not None:
            self._owner._columns = None

    # -- metadata -------------------------------------------------------------------------
    def _check(self):
        assert self._name is not None, "null Read"

    name = property(lambda self: (self._check(), self._name)[1])
    mapqs = property(lambda self: (self._check(), tuple(self._mapqs))[1])
    source_id = property(lambda self: (self._check(), self._source_id)[1])
    sample_id = property(lambda self: (self._check(), self._sample_id)[1])
    reference_start = property(lambda self: (self._check(), self._reference_start)[1])
    reference_end = property(lambda self: (self._check(), self._reference_end)[1])
    chromosome = property(lambda self: (self._check(), self._chromosome)[1])
    sub_alignment_id = property(lambda self: (self._check(), self._sub_alignment_id)[1])
    is_supplementary = property(lambda self: (self._check(), self._is_supplementary)[1])
    is_reverse = property(lambda self: (self._check(), self._is_reverse)[1])
    BX_tag = property(lambda self: (self._check(), self._BX_tag)[1])
    HP_tag = property(lambda self: (self._check(), self._HP_tag)[1])
    PS_tag = property(lambda self: (self._check(), self._PS_tag)[1])

    def __repr__(self):
        self._check()
        return (
            "Read(name={!r}, mapq={}, source_id={}, sample_id={}, reference_start={}, reference_end={}, chromosome={}, "
            "is_supplementary={}, is_reverse={},  BX_tag={}, HP_tag={}, PS_tag={}, variants={})".format(
                self.name, self.mapqs, self.source_id, self.sample_id, self.reference_start, self.reference_end,
                self.chromosome, self.is_supplementary, self.is_reverse, self.BX_tag, self.HP_tag, self.PS_tag, list(self),
            )
        )

    # -- variants -------------------------------------------------------------------------
    def __iter__(self) -> Iterator[Variant]:
        self._check()
        for i in range(len(self._pos)):
            yield self[i]

    def __len__(self):
        self._check()
        return len(self._pos)

    def __getitem__(self, key) -> Variant:
        self._check()
        if isinstance(key, slice):
            raise NotImplementedError("Read does not support slices")
        assert isinstance(key, int)
        n = len(self._pos)
        if not (-n <= key < n):
            raise IndexError("Index out of bounds: {}".format(key))
        if key < 0:
            key += n
        return Variant(position=self._pos[key], allele=self._allele[key], quality=self._quality[key])

    def __setitem__(self, index, variant):
        self._check()
        n = len(self._pos)
        if not (-n <= index < n):
            raise IndexError("Index out of bounds: {}".format(index))
        if index < 0:
            index += n
        if not isinstance(variant, Variant):
            raise ValueError("Expected instance of Variant, but found {}".format(type(variant)))
        self._pos[index] = int(variant.position)
        self._allele[index] = int(variant.allele)
        self._quality[index] = int(variant.quality)
        self._touch()

    def __contains__(self, position):
        self._check()
        assert isinstance(position, int)
        return position in self._pos

    def add_variant(self, position: int, allele: int, quality: int):
        self._check()
        self._pos.append(int(position))
        self._allele.append(int(allele))
        self._quality.append(int(quality))
        if self._owner is not None:
            self._owner._columns = None

    def add_mapq(self, mapq: int):
        self._check()
        self._mapqs.append(int(mapq))

    def sort(self):
        """Sort variants by position; duplicates raise like Read::sortVariants (src/read.cpp:66-75)."""
        self._check()
        order = sorted(range(len(self._pos)), key=self._pos.__getitem__)  # stable, like std::sort on distinct keys
        self._pos = array("q", [self._pos[i] for i in order])
        self._allele = array("q", [self._allele[i] for i in order])
        self._quality = array("q", [self._quality[i] for i in order])
        self._touch()
        for i in range(1, len(self._pos)):
            if self._pos[i - 1] == self._pos[i]:
                raise RuntimeError("Duplicate variant in read {} at position {}".format(self._name, self._pos[i]))

    def is_sorted(self):
        self._check()
        p = self._pos
        return all(p[i - 1] < p[i] for i in range(1, len(p)))

    def has_BX_tag(self):
        self._check()
        return self._BX_tag != ""

    # the reference answers all three questions with hasBXTag() (core.pyx:263-273); kept as is
    has_HP_tag = has_BX_tag
    has_PS_tag = has_BX_tag

    # -- copying / pickling ---------------------------------------------------------------
    def _clone(self) -> "Read":
        r = Read.__new__(Read)
        for slot in Read.__slots__:
            v = getattr(self, slot)
            setattr(r, slot, list(v) if isinstance(v, list) else (array("q", v) if isinstance(v, array) else v))
        r._owner = None
        return r

    def __getstate__(self):
        variants = [(p, a, q) for p, a, q in zip(self._pos, self._allele, self._quality)]
        return (list(self._mapqs), self._name, self._source_id, self._sample_id, self._reference_start,
                self._reference_end, self._BX_tag, self._HP_tag, self._PS_tag, self._chromosome, self._sub_alignment_id,
                self._is_supplementary, self._is_reverse, variants)

    def __setstate__(self, state):
        (mapqs, name, source_id, sample_id, reference_start, reference_end, BX_tag, HP_tag, PS_tag, chromosome,
         sub_alignment_id, is_supplementary, is_reverse, variants) = state
        Read.__init__(self, name, mapqs[0] if mapqs else 0, source_id, sample_id, reference_start, BX_tag, HP_tag, PS_tag,
                      chromosome, sub_alignment_id, is_supplementary, reference_end, is_reverse)
        for mapq in mapqs[1:]:
            self.add_mapq(mapq)
        for pos, allele, quality in variants:
            self.add_variant(pos, allele, quality)


class ReadSet:
    """Ordered collection of reads (core.pyx:275-361, src/readset.cpp)."""

    def __init__(self):
        self._reads: List[Read] = []
        self._by_name: Dict[Tuple[str, int], int] = {}
        # Columnar copy of all variants in read order: [lens, sample ids, positions, alleles, qualities] as array('q').  The
        # reference's ReadSet copies every added read into one C++ container that the DP then walks in place; here `add` appends
        # the read's three typed arrays to the set's (memcpy), so that `_flatten_reads` starts from five flat arrays instead of
        # visiting 50k Python objects.  None = stale (a stored read was changed through a reference): rebuilt on demand.
        self._columns = [array("q"), array("q"), array("q"), array("q"), array("q")]

    def add(self, read: Read):
        """Adds a COPY of the read (core.pyx:282-287); duplicate (name, source_id) raises
        (src/readset.cpp:22-29)."""
        key = (read.name, read.source_id)
        if key in self._by_name:
            raise RuntimeError("ReadSet::add: duplicate read name.")
        self._by_name[key] = len(self._reads)
        clone = read._clone()
        clone._owner = self
        self._reads.append(clone)
        cols = self._columns
        if cols is not None:
            cols[0].append(len(clone._pos))
            cols[1].append(clone._sample_id)
            cols[2].extend(clone._pos)
            cols[3].extend(clone._allele)
            cols[4].extend(clone._quality)

    def _flat_columns(self):
        """(lens, sample ids, positions, alleles, qualities) of all reads as int64 numpy arrays (copies)."""
        cols = self._columns
        if cols is None:  # a stored read was modified: collect again from the objects
            reads = self._reads
            cols = [array("q", (len(r._pos) for r in reads)), array("q", (r._sample_id for r in reads)), array("q"), array("q"), array("q")]
            cols[2].frombytes(b"".join(r._pos for r in reads))
            cols[3].frombytes(b"".join(r._allele for r in reads))
            cols[4].frombytes(b"".join(r._quality for r in reads))
            self._columns = cols
        return tuple(np.array(c, np.int64) for c in cols)

    def __str__(self):
        lines = ["ReadSet:"]
        for i, r in enumerate(self._reads):
            mapqs = ",".join(str(q) for q in r._mapqs)
            variants = ";".join(
                "[{},Entry({},{},{})]".format(p, 0, {0: "REF", 1: "ALT", 2: "BLANK", 3: "EQUAL_SCORES"}.get(a, a), q)
                for p, a, q in zip(r._pos, r._allele, r._quality)
            )
            lines.append("  {:>5} {} mapq:({}) source:{} sample:{} ({})".format(i, r._name, mapqs, r._source_id, r._sample_id, variants))
        return "\n".join(lines) + "\n"

    def __iter__(self):
        for i in range(len(self._reads)):
            yield self._reads[i]

    def __len__(self):
        return len(self._reads)

    def __getitem__(self, key):
        if isinstance(key, slice):
            raise NotImplementedError("ReadSet does not support slices")
        if isinstance(key, int):
            return self._reads[key]
        if isinstance(key, str):
            raise NotImplementedError(
                "Querying a ReadSet by read name is deprecated, please query by (source_id, name) instead"
            )
        if isinstance(key, tuple) and len(key) == 2 and isinstance(key[0], int) and isinstance(key[1], str):
            idx = self._by_name.get((key[1], key[0]))
            if idx is None:
                raise KeyError(key)
            return self._reads[idx]
        assert False, "Invalid key: {}".format(key)

    def __getstate__(self):
        return [read for read in self]

    def __setstate__(self, state):
        self.__init__()
        for read in state:
            self.add(read)

    def sort(self):
        """Sort by position of the first variant; reads without variants first; ties by
        libstdc++'s hash of (name, source_id), then name, then source_id — the exact order of
        ReadSet::read_comparator_t (src/readset.h:39-66), because read order defines the bit
        positions of the DP's bipartition indices."""

        def key(r: Read):
            first = r._pos[0] if r._pos else -1
            return (len(r._pos) > 0, first, _lib.read_sort_key(r._name, r._source_id), r._name.encode("utf-8"), r._source_id)

        order = sorted(range(len(self._reads)), key=lambda i: key(self._reads[i]))  # stable, like list.sort
        cols = self._columns
        if cols is not None and order != list(range(len(order))):
            # reorder the columnar copy with the same permutation (vectorised gather)
            lens, samples, pos, allele, quality = (np.array(c, np.int64) for c in cols)
            perm = np.array(order, np.int64)
            off = np.zeros(len(lens) + 1, np.int64)
            np.cumsum(lens, out=off[1:])
            new_lens = lens[perm]
            new_off = np.zeros(len(lens) + 1, np.int64)
            np.cumsum(new_lens, out=new_off[1:])
            idx = np.repeat(off[:-1][perm] - new_off[:-1], new_lens) + np.arange(int(new_off[-1]), dtype=np.int64)
            self._columns = [_typed(new_lens), _typed(samples[perm]), _typed(pos[idx]), _typed(allele[idx]), _typed(quality[idx])]
        self._reads = [self._reads[i] for i in order]
        self._by_name = {(r._name, r._source_id): i for i, r in enumerate(self._reads)}

    def subset(self, reads_to_select: Iterable[int]) -> "ReadSet":
        """Copies of the selected reads in ascending index order (IndexSet is a std::set, src/indexset.h)."""
        result = ReadSet()
        for i in sorted(set(int(i) for i in reads_to_select)):
            result.add(self._reads[i])
        return result

    def get_positions(self) -> List[int]:
        return _distinct_sorted(self._flat_columns()[2]).tolist()


class Genotype:
    """Unordered multiset of alleles (core.pyx:511-570, src/genotype.cpp)."""

    __slots__ = ("_alleles",)

    def __init__(self, alleles: Sequence[int]):
        alleles = [int(a) for a in alleles]
        if len(alleles) >= MAX_GENOTYPE_PLOIDY:
            raise RuntimeError("Error: Maximum ploidy for genotype exceeded!")
        for a in alleles:
            if a < 0:
                raise OverflowError("can't convert negative value to uint32_t")
            if a >= MAX_GENOTYPE_ALLELES:
                raise RuntimeError("Error: Maximum alleles for genotype exceeded!")
        self._alleles = tuple(sorted(alleles))

    def __str__(self):
        if self.is_none():
            return "."
        return "/".join(str(a) for a in self._alleles)

    __repr__ = __str__

    def is_none(self):
        return len(self._alleles) == 0

    def get_index(self) -> int:
        """Canonical VCF index (src/genotype.cpp:82-93)."""
        index, k = 0, 1
        for allele in self._alleles:
            index += comb(k + allele - 1, allele - 1) if allele >= 1 else 0
            k += 1
        return index

    def as_vector(self) -> List[int]:
        # the reference stores the highest allele in the lowest nibble and reads nibbles upwards
        return list(reversed(self._alleles))

    def is_homozygous(self):
        return (not self.is_none()) and len(set(self._alleles)) == 1

    def is_diploid_and_biallelic(self):
        return len(self._alleles) == 2 and all(a <= 1 for a in self._alleles)

    def get_ploidy(self):
        return len(self._alleles)

    def __eq__(self, g):
        return isinstance(g, Genotype) and self._alleles == g._alleles

    def __ne__(self, g):
        return not self.__eq__(g)

    def __lt__(self, g):
        return self.get_index() < g.get_index()

    def __getstate__(self):
        return (self.get_index(), self.get_ploidy())

    def __setstate__(self, state):
        index, ploidy = state
        self._alleles = tuple(sorted(_index_to_alleles(index, ploidy)))

    def __deepcopy__(self, memo):
        return Genotype(list(self._alleles))

    def __hash__(self):
        return hash(self.get_index())


def _index_to_alleles(index: int, ploidy: int) -> List[int]:
    """Inverse of Genotype.get_index for a given ploidy (enumeration of sorted allele multisets)."""
    alleles = []
    remaining = index
    for p in range(ploidy, 0, -1):
        a = 0
        while comb(p + a, p) <= remaining:  # number of multisets of size p over alleles 0..a
            a += 1
        remaining -= comb(p + a - 1, p)
        alleles.append(a)
    return alleles


def get_max_genotype_ploidy():
    return MAX_GENOTYPE_PLOIDY


def get_max_genotype_alleles():
    return MAX_GENOTYPE_ALLELES


def binomial_coefficient(n: int, k: int) -> int:
    if k < 0 or n < 0 or n < k:
        return 0
    return comb(n, k)


class PhredGenotypeLikelihoods:
    """Phred-scaled genotype likelihoods indexed by canonical genotype index (core.pyx:469-504)."""

    def __init__(self, gl: Sequence[float], ploidy: int = 2, nr_alleles: int = 2):
        self._gl = [float(x) for x in gl]
        self._ploidy = int(ploidy)
        self._nr_alleles = int(nr_alleles)
        if binomial_coefficient(self._ploidy + self._nr_alleles - 1, self._nr_alleles - 1) != len(self._gl):
            raise RuntimeError("Error: wrong number of given genotype likelihoods given.")

    def __str__(self):
        def fmt(x):
            return str(int(x)) if x == int(x) else repr(x)

        return "PhredGenotypeLikelihoods(" + ",".join(fmt(x) for x in self._gl)

    def __getitem__(self, genotype: Genotype):
        assert genotype.is_diploid_and_biallelic()
        assert self._ploidy == genotype.get_ploidy()
        return self._gl[genotype.get_index()]

    def __len__(self):
        return len(self._gl)

    def __iter__(self):
        for genotype in self.genotypes():
            yield self[genotype]

    def __eq__(self, other):
        if self.genotypes() != other.genotypes():
            return False
        return all(self[g] == other[g] for g in self.genotypes())

    def genotypes(self) -> List[Genotype]:
        return [Genotype(_index_to_alleles(i, self._ploidy)) for i in range(len(self._gl))]

    def as_vector(self):
        return list(self._gl)

    def get_ploidy(self):
        return self._ploidy

    def get_nr_alleles(self):
        return self._nr_alleles


_GT_CODE = {(0, 0): 0, (0, 1): 1, (1, 1): 2}


class Pedigree:
    """Individuals with per-variant genotypes (and likelihoods) plus trio relationships
    (core.pyx:419-466, src/pedigree.cpp)."""

    def __init__(self, numeric_sample_ids: NumericSampleIds):
        self.numeric_sample_ids = numeric_sample_ids
        self._ids: List[int] = []
        self._index: Dict[int, int] = {}
        self._genotypes: List[List[Genotype]] = []
        self._gt_codes: List[np.ndarray] = []
        self._gls: List[List[Optional[PhredGenotypeLikelihoods]]] = []
        self._triples: List[Tuple[int, int, int]] = []
        self._variant_count = -1

    def add_individual(self, id, genotypes, genotype_likelihoods=None):
        gts = []
        for gt in genotypes:
            if not isinstance(gt, Genotype):
                raise TypeError("Cannot convert {} to Genotype".format(type(gt).__name__))
            gts.append(copy.deepcopy(gt))
        if genotype_likelihoods:
            gls = []
            for gl in genotype_likelihoods:
                if gl is not None and not isinstance(gl, PhredGenotypeLikelihoods):
                    raise TypeError("Cannot convert {} to PhredGenotypeLikelihoods".format(type(gl).__name__))
                gls.append(gl)
        else:
            gls = [None] * len(gts)
        if self._variant_count == -1:
            self._variant_count = len(gts)
        assert len(gts) == self._variant_count
        assert len(gls) == self._variant_count
        numeric = self.numeric_sample_ids[id]
        # canonical index of the diploid biallelic genotypes (genotype.cpp:82-93) as one byte per variant, for `_flatten`
        self._gt_codes.append(np.fromiter((_GT_CODE.get(g._alleles, GT_OTHER) for g in gts), np.uint8, count=len(gts)))
        self._genotypes.append(gts)
        self._gls.append(gls)
        self._ids.append(numeric)
        self._index[numeric] = len(self._ids) - 1

    def add_relationship(self, father_id, mother_id, child_id):
        self._triples.append(
            (self.id_to_index(self.numeric_sample_ids[father_id]), self.id_to_index(self.numeric_sample_ids[mother_id]),
             self.id_to_index(self.numeric_sample_ids[child_id]))
        )

    def id_to_index(self, numeric_id: int) -> int:
        if numeric_id not in self._index:
            raise RuntimeError("Individual with ID {} not present in pedigree.".format(numeric_id))
        return self._index[numeric_id]

    def index_to_id(self, index: int) -> int:
        return self._ids[index]

    @property
    def variant_count(self):
        """Number of variants stored for each individual."""
        return self._variant_count

    def genotype(self, sample_id, variant_index: int) -> Genotype:
        gt = self._genotypes[self.id_to_index(self.numeric_sample_ids[sample_id])][variant_index]
        return Genotype(gt.as_vector())

    def genotype_likelihoods(self, sample_id, variant_index: int):
        gl = self._gls[self.id_to_index(self.numeric_sample_ids[sample_id])][variant_index]
        if gl is None:
            return None
        return PhredGenotypeLikelihoods(gl.as_vector(), gl.get_ploidy(), gl.get_nr_alleles())

    def __len__(self):
        return len(self._ids)

    def __str__(self):
        out = ["Pedigree:"]
        out.append("  individuals (index,id):" + "".join(" {},{}".format(i, d) for i, d in enumerate(self._ids)))
        out.append("  triples by index (father,mother,child):" + "".join(" ({},{},{})".format(*t) for t in self._triples))
        out.append("  triples by id (father,mother,child):" + "".join(
            " ({},{},{})".format(self._ids[t[0]], self._ids[t[1]], self._ids[t[2]]) for t in self._triples))
        out.append("  genotypes (and likelihoods):")
        for i, d in enumerate(self._ids):
            out.append("    individual index:{} / id:{}:".format(i, d))
            for j in range(max(self._variant_count, 0)):
                gl = self._gls[i][j]
                out.append("      {} (GL:{}".format(self._genotypes[i][j], "None)" if gl is None else str(gl)))
        return "\n".join(out) + "\n"


def _flatten_reads(readset: ReadSet, positions: Optional[Sequence[int]], index_of_sample):
    """The read side of `_flatten`: (pos_list, read_off, ent_col, ent_allele, ent_phred, read_ind).
    `index_of_sample(sample_id)` gives the pedigree index of a read's sample."""
    reads = readset._reads
    m = len(reads)
    lens, samples, pos, allele, quality = readset._flat_columns()
    if positions is None:
        pos_arr = _distinct_sorted(pos)
        pos_list = pos_arr.tolist()
    else:
        pos_list = [int(p) for p in positions]
        pos_arr = np.array(pos_list, np.int64)
    n = len(pos_list)
    # sample id -> pedigree index, once per distinct sample (raises like id_to_index for an unknown one)
    if m:
        uniq, first_at, inverse = np.unique(samples, return_index=True, return_inverse=True)
        index_of = np.zeros(len(uniq), np.uint32)
        for u in np.argsort(first_at, kind="stable"):  # in read order: the first read with an unknown sample raises
            index_of[u] = index_of_sample(int(uniq[u]))
        read_ind = index_of[inverse]
    else:
        read_ind = np.zeros(0, np.uint32)
    if m and int(lens.min()) == 0:
        raise RuntimeError("No variants present")
    total = int(lens.sum())
    off = np.zeros(m + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    if m:
        first, last_i = off[:-1], off[1:] - 1
        if m > 1 and bool((np.diff(pos[first]) < 0).any()):
            raise RuntimeError("ColumnIterator: reads in ReadSet are not sorted.")
        step = np.diff(pos)
        step[last_i[:-1]] = 1  # differences across read boundaries do not count
        if bool((step <= 0).any()):
            raise RuntimeError("ColumnIterator: encountered read with unsorted variants.")
    if n and bool((np.diff(pos_arr) <= 0).any()):
        # unsorted / repeated explicit positions: the last occurrence defines the column, as in a dict
        col_of = {p: i for i, p in enumerate(pos_list)}
        col = np.fromiter((col_of.get(int(p), -1) for p in pos), np.int64, count=total)
    elif n and int(pos_arr[-1]) - int(pos_arr[0]) <= 16 * n + 1024:
        # densely numbered positions: a look-up table over the position range instead of a binary search per entry
        lo_p, hi_p = int(pos_arr[0]), int(pos_arr[-1])
        lut = np.full(hi_p - lo_p + 1, -1, np.int64)
        lut[pos_arr - lo_p] = np.arange(n, dtype=np.int64)
        inside = (pos >= lo_p) & (pos <= hi_p)
        col = np.where(inside, lut[np.clip(pos, lo_p, hi_p) - lo_p], -1)
    elif n and positions is None:
        # every position of a read is a column.  Reads mostly cover consecutive columns: one binary search per READ, then
        # column = first column + offset inside the read wherever the position found there is the entry's, and a binary search
        # only for the entries behind a gap
        first_col = np.searchsorted(pos_arr, pos[off[:-1]]) if m else np.zeros(0, np.int64)
        col = np.repeat(first_col - off[:-1], lens) + np.arange(total, dtype=np.int64)
        np.minimum(col, n - 1, out=col)
        behind_gap = np.nonzero(pos_arr[col] != pos)[0]
        if behind_gap.size:
            col[behind_gap] = np.searchsorted(pos_arr, pos[behind_gap])
    elif n:
        col = np.searchsorted(pos_arr, pos)
        col = np.where((col < n) & (pos_arr[np.minimum(col, n - 1)] == pos), col, -1)
    else:
        col = np.full(total, -1, np.int64)
    all_valid = bool(n) and (positions is None or int(col.min(initial=0)) >= 0)
    valid = None if all_valid else col >= 0
    if m and not all_valid:
        bad = np.nonzero(~(valid[first] & valid[last_i]))[0]
        if bad.size:
            # the reference asserts here (columniterator.cpp:36-39) and aborts the process
            raise RuntimeError("read {!r}: first/last variant position is not among the given positions".format(reads[int(bad[0])].name))
    # interior variants outside `positions` are skipped (columniterator.cpp:101-104)
    if total and (int(allele.min()) < 0 or int(allele.max()) > 2):
        outside = (allele < 0) | (allele > 2)
        wrong = np.nonzero(outside if all_valid else (valid & outside))[0]
        if wrong.size:
            r_idx = int(np.searchsorted(off, wrong[0], side="right") - 1)
            raise RuntimeError("read {!r}: allele {} is not 0 (REF), 1 (ALT) or 2 (BLANK)".format(reads[r_idx].name, int(allele[wrong[0]])))
    if total and int(quality.min()) < 0 and bool(((quality < 0) if all_valid else (valid & (quality < 0))).any()):
        raise OverflowError("negative quality")
    read_off = np.zeros(m + 1, np.uint64)
    if all_valid:
        read_off[1:] = off[1:]
        return pos_list, read_off, col, allele, quality, read_ind
    kept = np.add.reduceat(valid.astype(np.int64), off[:-1]) if m else np.zeros(0, np.int64)
    np.cumsum(kept, out=read_off[1:])
    return pos_list, read_off, col[valid], allele[valid], quality[valid], read_ind


def _flatten(readset: ReadSet, recombcost: Sequence[int], pedigree: Pedigree, distrust_genotypes: bool,
             positions: Optional[Sequence[int]]) -> FlatProblem:
    """ReadSet / Pedigree / recombcost -> the CSR arrays of `whmec_problem` (include/whmec.h).

    Restates the input side of the reference constructor: `reassignReadIds`, the sample-id to
    pedigree-index translation (src/pedigreedptable.cpp:24-34) and ColumnIterator's mapping of
    positions to columns (src/columniterator.cpp:12-22)."""
    pos_list, read_off, ent_col, ent_allele, ent_phred, read_ind = _flatten_reads(readset, positions, pedigree.id_to_index)
    n = len(pos_list)
    # -- pedigree --------------------------------------------------------------------------------------
    n_ind = len(pedigree)
    if n_ind == 0:
        raise RuntimeError("pedigree without individuals")
    if n > 0 and pedigree.variant_count != -1 and pedigree.variant_count < n:
        raise RuntimeError("pedigree holds genotypes for {} variants but the DP has {} columns".format(pedigree.variant_count, n))
    rc = recombcost.tolist() if isinstance(recombcost, np.ndarray) else [int(x) for x in recombcost]
    if len(rc) < n:
        # The reference indexes recombcost[column] without a bounds check (pedigreedptable.cpp:291) and
        # its own tests pass lists that are one short (tests/test_pedigreephasing.py:247,266); reading
        # past the end is undefined there, here the last given cost is repeated.
        rc = rc + [rc[-1] if rc else 0] * (n - len(rc))
    gt = np.full((n_ind, n), GT_OTHER, np.uint8)
    gl = np.zeros((n_ind, n, 3), np.float64) if distrust_genotypes else None
    for i in range(n_ind):
        gt[i, :] = pedigree._gt_codes[i][:n]
        if distrust_genotypes:
            for k in range(n):
                lk = pedigree._gls[i][k]
                if lk is None:
                    # assert(gls != nullptr) in the reference (pedigreecolumncostcomputer.cpp:36)
                    raise RuntimeError("distrust_genotypes requires genotype likelihoods for every variant")
                if lk.get_ploidy() != 2:
                    raise RuntimeError("genotype likelihoods must be diploid")
                gl[i, k, :] = lk._gl[:3]
    trios = [x for t in pedigree._triples for x in t]
    return FlatProblem(
        positions=np.array(pos_list, np.uint32),
        read_off=np.array(read_off, np.uint64),
        ent_col=np.array(ent_col, np.uint32),
        ent_allele=np.array(ent_allele, np.uint8),
        ent_phred=np.array(ent_phred, np.uint32),
        read_ind=np.array(read_ind, np.uint32),
        recombcost=np.array(rc[:n], np.uint32),
        n_ind=n_ind,
        trios=np.array(trios, np.uint32),
        distrust=bool(distrust_genotypes),
        gt=gt,
        gl=gl,
    )


class PedigreeDPTable:
    """Exact weighted-MEC / PedMEC solver; the constructor does all the work
    (core.pyx:364-416; abstract contract whatshap/types.py:7-15).  `devices` (CUDA ordinals; default: those of
    WHMEC_DEVICES if it is set) spreads the table over several GPUs from this process (`multigpu.solve_on_devices`) with
    the same result; otherwise it runs on `device`."""

    def __init__(self, readset: ReadSet, recombcost, pedigree: Pedigree, distrust_genotypes: bool = False,
                 positions=None, device: int = 0, devices=None):
        if not isinstance(readset, ReadSet):
            raise TypeError("Argument 'readset' has incorrect type")
        if not isinstance(pedigree, Pedigree):
            raise TypeError("Argument 'pedigree' has incorrect type")
        self.pedigree = pedigree
        self._problem = _flatten(readset, recombcost, pedigree, bool(distrust_genotypes), positions)
        self._solution, self.stats = multigpu.solve_table(self._problem, device, devices)

    @classmethod
    def batch(cls, tables, device: int = 0, devices=None, return_exceptions: bool = False) -> list:
        """Several tables in one call, sharing the GPU (`multigpu.solve_tables`, `whmec_solve_batch`).  `tables` is a sequence of
        constructor argument tuples `(readset, recombcost, pedigree[, distrust_genotypes[, positions]])`; every returned object
        behaves exactly like `cls(*arguments)`.  A table that fails does not stop the others: afterwards the error of the
        lowest-index failing table is raised, with the type and text the constructor would have raised; with
        `return_exceptions` the exception instance takes the table's place instead."""
        def build(obj, args):
            readset, recombcost, pedigree = args[0], args[1], args[2]
            if not isinstance(readset, ReadSet):
                raise TypeError("Argument 'readset' has incorrect type")
            if not isinstance(pedigree, Pedigree):
                raise TypeError("Argument 'pedigree' has incorrect type")
            obj.pedigree = pedigree
            obj._problem = _flatten(readset, recombcost, pedigree, bool(args[3]) if len(args) > 3 else False, args[4] if len(args) > 4 else None)
            obj.stats = {}

        return multigpu.batch_objects(cls, tables, build, lambda problems: multigpu.solve_tables(problems, device, devices, with_stats=True),
                                      "_solution", return_exceptions)

    def get_super_reads(self) -> Tuple[List[ReadSet], List[int]]:
        """One ReadSet per individual (pedigree order) holding `superread_0_<k>` and
        `superread_1_<k>`, plus the transmission vector (src/pedigreedptable.cpp:344-388)."""
        prob, sol = self._problem, self._solution
        results = []
        positions = prob.positions
        for k in range(len(self.pedigree)):
            rs = ReadSet()
            quality = sol.sr_quality[k]
            for h in range(2):
                read = Read("superread_{}_{}".format(h, k), -1, -1, self.pedigree.index_to_id(k))
                read._pos = _typed(positions)
                read._allele = _typed(sol.sr_allele[k, h])
                read._quality = _typed(quality)
                rs.add(read)
            results.append(rs)
        return results, sol.path_tv.tolist()

    def get_optimal_cost(self) -> int:
        """MEC score; declared `int` in the reference binding (cpp.pxd:89)."""
        c = int(self._solution.cost)
        return c - (1 << 32) if c >= (1 << 31) else c

    def get_optimal_partitioning(self) -> List[int]:
        return self._solution.partition.tolist()


class PedMecHeuristic:
    """Row-limited heuristic PedMEC solver, `whatshap phase --algorithm=heuristic` (core.pyx:674-734, src/pedmecheuristic.cpp).

    Same constructor and methods as the reference binding.  Unlike `PedigreeDPTable` one table is HOST code (`whmec_heuristic`,
    csrc/heuristic.cpp): a sequential beam search over float scores whose results equal the reference's bit for bit.  Many tables
    go to the GPU together through `batch` (one CTA per table, the same results).
    The reads' sample ids must be the zero-based indices of the pedigree's individuals (src/pedmecheuristic.h:66)."""

    def __init__(self, readset: ReadSet, recombcost, pedigree: Pedigree, row_limit: int = 256, distrust_genotypes: bool = False,
                 positions=None, allow_mutations: bool = True, verbosity: int = 0):
        self._setup(readset, recombcost, pedigree, distrust_genotypes, positions)
        self._solution = _lib.heuristic(self._problem, min(max(int(row_limit), 0), 65535), bool(allow_mutations))

    def _setup(self, readset, recombcost, pedigree, distrust_genotypes, positions) -> None:
        """The constructor's checks and its flat problem (`_problem`), before the solver runs."""
        if not isinstance(readset, ReadSet):
            raise TypeError("Argument 'readset' has incorrect type")
        if not isinstance(pedigree, Pedigree):
            raise TypeError("Argument 'pedigree' has incorrect type")
        self.pedigree = pedigree
        n_ind = len(pedigree)

        def sample_index(sample_id: int) -> int:
            if not 0 <= sample_id < n_ind:
                raise RuntimeError("PedMecHeuristic: sample id {} is not a zero-based index into the pedigree".format(sample_id))
            return sample_id

        pos_list, read_off, ent_col, ent_allele, ent_phred, read_ind = _flatten_reads(readset, positions, sample_index)
        n = len(pos_list)
        if n_ind == 0:
            raise RuntimeError("pedigree without individuals")
        if n > 0 and pedigree.variant_count != -1 and pedigree.variant_count < n:
            raise RuntimeError("pedigree holds genotypes for {} variants but there are {} columns".format(pedigree.variant_count, n))
        rc = [int(x) for x in recombcost]
        if len(rc) < n:
            rc = rc + [rc[-1] if rc else 0] * (n - len(rc))
        gt = np.full((n_ind, n), GT_OTHER, np.uint8)
        for i in range(n_ind):
            gt[i, :] = pedigree._gt_codes[i][:n]
        self._problem = FlatProblem(
            positions=np.array(pos_list, np.uint32), read_off=np.array(read_off, np.uint64), ent_col=np.array(ent_col, np.uint32),
            ent_allele=np.array(ent_allele, np.uint8), ent_phred=np.array(ent_phred, np.uint32), read_ind=np.array(read_ind, np.uint32),
            recombcost=np.array(rc[:n], np.uint32), n_ind=n_ind, trios=np.array([x for t in pedigree._triples for x in t], np.uint32),
            distrust=bool(distrust_genotypes), gt=gt, gl=None)
        # the samples the solver knows: ids of the reads and of the trio members, ascending (pedmecheuristic.cpp:52-63)
        self._sample_ids = sorted(set(self._problem.read_ind.tolist()) | set(self._problem.trios.tolist()))

    @classmethod
    def batch(cls, tables, device: int = 0, devices=None, return_exceptions: bool = False) -> list:
        """Several tables in one call, one CTA of the GPU per table (`multigpu.heuristic_tables`, `whmec_heuristic_batch`).  `tables`
        is a sequence of constructor argument tuples `(readset, recombcost, pedigree[, row_limit[, distrust_genotypes[, positions[,
        allow_mutations[, verbosity]]]]])`; every returned object answers exactly like `cls(*arguments)`.  A table that fails does
        not stop the others: afterwards the error of the lowest-index failing table is raised, with the type and text the
        constructor would have raised; with `return_exceptions` the exception instance takes the table's place instead."""
        def setup(obj, args):
            obj._setup(args[0], args[1], args[2], args[4] if len(args) > 4 else False, args[5] if len(args) > 5 else None)

        return multigpu.batch_heuristic_objects(cls, tables, setup, device, devices, return_exceptions)

    def get_super_reads(self) -> Tuple[List[ReadSet], List[int]]:
        """One ReadSet per sample with `superread_0` / `superread_1` (quality 30 everywhere, pedmecheuristic.cpp:104-117),
        plus the transmission vector."""
        prob, sol = self._problem, self._solution
        results = []
        quality = np.full(prob.n_cols, 30, np.int64)
        for k, sid in enumerate(self._sample_ids):
            rs = ReadSet()
            for h in range(2):
                read = Read("superread_{}".format(h), -1, -1, sid)
                read._pos = _typed(prob.positions)
                read._allele = _typed(sol.haplotypes[k, h].astype(np.int64))
                read._quality = _typed(quality)
                rs.add(read)
            results.append(rs)
        return results, sol.transmission.tolist()

    def get_optimal_cost(self) -> float:
        """The reference's getOptScore(): a member its solve() never assigns, i.e. always 0.0 (pedmecheuristic.cpp:84-86)."""
        return float(self._solution.score)

    def get_optimal_partitioning(self) -> List[int]:
        return [0 if x else 1 for x in self._solution.partition.tolist()]  # core.pyx:719

    def get_mutations(self) -> List[List[Tuple[int, int]]]:
        """Per sample the (haplotype, column) pairs whose allele does not follow the parent (core.pyx:722-734)."""
        sol = self._solution
        out = []
        for k in range(sol.n_samples):
            cols, haps = np.nonzero(sol.mutated[k].T)  # column-major: per column haplotype 0 before 1
            out.append([(int(h), int(c)) for c, h in zip(cols, haps)])
        return out


class GenotypeDPTable:
    """Genotype likelihoods by the forward-backward algorithm over the same bipartition DP; the constructor
    does all the work (core.pyx:581-600, src/genotypedptable.cpp:17-48).  `pedigree` must carry genotype
    likelihoods (priors) for every variant; `recombcost` are phred-scaled recombination probabilities.  `device` /
    `devices` as for `PedigreeDPTable` (`multigpu.genotype_on_devices`)."""

    def __init__(self, numeric_sample_ids: NumericSampleIds, readset: ReadSet, recombcost, pedigree: Pedigree,
                 positions=None, device: int = 0, devices=None):
        if not isinstance(readset, ReadSet):
            raise TypeError("Argument 'readset' has incorrect type")
        if not isinstance(pedigree, Pedigree):
            raise TypeError("Argument 'pedigree' has incorrect type")
        self.pedigree = pedigree
        self.numeric_sample_ids = numeric_sample_ids
        # the priors travel in the `gl` array of the flat problem (as they do for distrusted genotypes)
        self._problem = _flatten(readset, recombcost, pedigree, True, positions)
        self._likelihoods, self.stats = multigpu.genotype_table(self._problem, device, devices)

    @classmethod
    def batch(cls, tables, device: int = 0, devices=None, return_exceptions: bool = False) -> list:
        """Several tables in one call, sharing the GPU's launches (`multigpu.genotype_tables`, `whmec_genotype_batch`).  `tables`
        is a sequence of constructor argument tuples `(numeric_sample_ids, readset, recombcost, pedigree[, positions])`; every
        returned object answers `get_genotype_likelihoods` exactly like `cls(*arguments)`.  A table that fails does not stop the
        others: afterwards the error of the lowest-index failing table is raised, with the type and text the constructor would
        have raised; with `return_exceptions` the exception instance takes the table's place instead."""
        def build(obj, args):
            numeric_sample_ids, readset, recombcost, pedigree = args[0], args[1], args[2], args[3]
            if not isinstance(readset, ReadSet):
                raise TypeError("Argument 'readset' has incorrect type")
            if not isinstance(pedigree, Pedigree):
                raise TypeError("Argument 'pedigree' has incorrect type")
            obj.pedigree = pedigree
            obj.numeric_sample_ids = numeric_sample_ids
            obj._problem = _flatten(readset, recombcost, pedigree, True, args[4] if len(args) > 4 else None)
            obj.stats = {}

        return multigpu.batch_objects(cls, tables, build, lambda problems: multigpu.genotype_tables(problems, device, devices, with_stats=True),
                                      "_likelihoods", return_exceptions)

    def get_genotype_likelihoods(self, sample_id, pos: int) -> PhredGenotypeLikelihoods:
        """Likelihoods of 0/0, 0/1, 1/1 of `sample_id` at column `pos` (src/genotypedptable.cpp:445-451)."""
        index = self.pedigree.id_to_index(self.numeric_sample_ids[sample_id])
        if not 0 <= pos < self._problem.n_cols:
            raise IndexError("position index out of range")  # assert in the reference
        return PhredGenotypeLikelihoods(self._likelihoods[index, pos].tolist())


def compute_genotypes(readset: ReadSet, positions=None):
    """Per-variant genotype priors from one sample's reads, the step `whatshap genotype` runs before `GenotypeDPTable`
    (core.pyx:602-617, src/genotyper.cpp:12-54): returns (genotypes, likelihoods) with `Genotype([])` where no genotype
    reaches an error probability below 0.1, and likelihoods as (hom-ref, het, hom-alt) tuples.  Host only; the doubles
    equal the reference's bit for bit."""
    if not isinstance(readset, ReadSet):
        raise TypeError("Argument 'readset' has incorrect type")
    pos_list, read_off, ent_col, ent_allele, ent_phred, read_ind = _flatten_reads(readset, positions, lambda sample: 0)
    n = len(pos_list)
    prob = FlatProblem(positions=np.array(pos_list, np.uint32), read_off=np.array(read_off, np.uint64), ent_col=np.array(ent_col, np.uint32),
                       ent_allele=np.array(ent_allele, np.uint8), ent_phred=np.array(ent_phred, np.uint32),
                       read_ind=np.array(read_ind, np.uint32), recombcost=np.zeros(n, np.uint32), n_ind=1)
    gl, gt = _lib.compute_genotypes(prob)
    genotypes = [Genotype(_index_to_alleles(int(g), 2)) if g >= 0 else Genotype([]) for g in gt.tolist()]
    return genotypes, [tuple(row) for row in gl.tolist()]
