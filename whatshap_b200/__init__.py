"""whatshap_b200 — CUDA (H100, sm_90a) weighted-MEC / PedMEC dynamic program behind WhatsHap's
`PedigreeDPTable` interface.  See DESIGN.md; the compute path is CUDA only (libwhmec.so)."""
from .core import (  # noqa: F401
    Genotype,
    GenotypeDPTable,
    NumericSampleIds,
    Pedigree,
    PedigreeDPTable,
    PedMecHeuristic,
    PhredGenotypeLikelihoods,
    Read,
    ReadSet,
    binomial_coefficient,
    compute_genotypes,
    get_max_genotype_alleles,
    get_max_genotype_ploidy,
)
from . import haplotag  # noqa: F401
from .learn import Caller, count_kmer_pairs, write_counts  # noqa: F401
from .types import PhasingAlgorithm  # noqa: F401
from .variant import Variant  # noqa: F401

PhasingAlgorithm.register(PedigreeDPTable)
PhasingAlgorithm.register(PedMecHeuristic)

__all__ = [
    "Genotype", "GenotypeDPTable", "NumericSampleIds", "Pedigree", "PedigreeDPTable", "PedMecHeuristic", "PhredGenotypeLikelihoods", "Read", "ReadSet",
    "Variant", "PhasingAlgorithm", "compute_genotypes", "Caller", "count_kmer_pairs", "write_counts", "haplotag",
]
