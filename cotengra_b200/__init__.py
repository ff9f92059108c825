"""cotengra_b200 -- H100-native executor for cotengra's sliced contraction trees.

The drop-in for ONE path of jcmgray/cotengra: ``ContractionTree.contract()`` ->
per-slice ``Contractor`` node loop -> pairwise tensordot/einsum
(cotengra/core.py:3943-4030, cotengra/contract.py:364-411, 718-837).  Tree
search, hyper-optimisation and slicing stay in cotengra, unchanged, on the host.

Importing this package does not need a GPU (planning is host-side integer
work); every compute entry point needs ``libctgb200.so`` and a CUDA device and
fails loudly otherwise.
"""

from .tree import TreeSpec, get_symbol
from .lowering import (
    PairDims,
    build_pair_desc,
    build_single_desc,
    classify_pair,
    classify_single,
)
from .executor import ExecPlan
from .jvp import JvpPlan
from .vjp import VjpPlan
from .contract import (
    B200Contractor,
    TreeExecutor,
    array_contract_expression,
    benchmark,
    contract_checkpointed,
    contract_distributed,
    contract_tree,
    einsum,
    gen_output_chunks,
    implementation,
    install,
    make_contractor,
    rank_slices,
    reduce_partials,
    tensordot,
)

__all__ = [
    "TreeSpec", "get_symbol", "PairDims", "build_pair_desc", "build_single_desc",
    "classify_pair", "classify_single", "ExecPlan", "VjpPlan", "JvpPlan", "B200Contractor", "TreeExecutor",
    "array_contract_expression", "benchmark", "contract_checkpointed", "contract_distributed", "contract_tree", "einsum", "gen_output_chunks", "implementation", "install",
    "make_contractor", "rank_slices", "reduce_partials", "tensordot",
]
