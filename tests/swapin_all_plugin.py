"""pytest plugin used by test_reference_suite_with_swapin.py (second run): the reference's test modules import
`whatshap.core`; before they do, EVERY class of this path in that module is replaced by this repository's Python
mirror (`whatshap_b200.core`), `whatshap.graph.ComponentFinder` by `whatshap_b200.components.ComponentFinder`, and the
CUDA solves behind `PedigreeDPTable` / `GenotypeDPTable` by the CPU checker (no GPU in the machine with the reference; the CUDA solve is held to the
same checker by the GPU tests).  The reference's tests then exercise this package's containers unmodified."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ["WHMEC_PYREF"])

import whatshap.core as core  # noqa: E402
import whatshap.graph  # noqa: E402
import whatshap.pedigree  # noqa: E402
import whatshap.priorityqueue  # noqa: E402
import whatshap.readselect  # noqa: E402
import whatshap.variant  # noqa: E402

import whatshap_b200 as mine  # noqa: E402
from oracle import checker  # noqa: E402
from whatshap_b200 import _lib, components  # noqa: E402
from whatshap_b200 import pedigree as my_pedigree  # noqa: E402
from whatshap_b200 import priorityqueue as my_queue  # noqa: E402
from whatshap_b200 import readselect as my_select  # noqa: E402

_checker = checker.port()
_lib.solve = lambda prob, device=0: (_checker.solve(prob), {})
import emul_genotype  # noqa: E402

_lib.genotype = emul_genotype.genotype  # the kernels' per-cell code + host packer, stepped on the host
for name in ("NumericSampleIds", "Read", "ReadSet", "Pedigree", "Genotype", "PhredGenotypeLikelihoods", "PedigreeDPTable", "GenotypeDPTable",
             "binomial_coefficient", "get_max_genotype_ploidy", "get_max_genotype_alleles"):
    setattr(core, name, getattr(mine, name) if hasattr(mine, name) else getattr(mine.core, name))
whatshap.graph.ComponentFinder = components.ComponentFinder
whatshap.variant.Variant = mine.Variant
if hasattr(core, "Variant"):
    core.Variant = mine.Variant
whatshap.readselect.readselection = my_select.readselection
whatshap.priorityqueue.PriorityQueue = my_queue.PriorityQueue
whatshap.pedigree.find_recombination = my_pedigree.find_recombination
whatshap.pedigree.centimorgen_to_phred = my_pedigree.centimorgen_to_phred
whatshap.pedigree.RecombinationEvent = my_pedigree.RecombinationEvent
# recombination costs fed to the pedigree / genotyping DP (tests/test_geneticmap.py of the reference)
for name in ("GeneticMapRecombinationCostComputer", "UniformRecombinationCostComputer", "ParseError", "recombination_cost_map", "mendelian_conflict"):
    if hasattr(my_pedigree, name) and hasattr(whatshap.pedigree, name):
        setattr(whatshap.pedigree, name, getattr(my_pedigree, name))
core.compute_genotypes = mine.compute_genotypes
