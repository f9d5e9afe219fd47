"""The marker-set reduction on a used workspace.  ckm_reduce and ckm_genome_check take their device buffers from the
engine's grow-only cache, which a search has just filled with its own data: the reduction must still match the
reference's goldens (tests/golden/reduction), so none of its kernels may read an element it has not written."""
import pytest

import test_reduction_gpu as reduction
from conftest import CPR_HMM
from test_reduction_gpu import golden, setup  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('case', ['kat1', 'stress'])
def test_reduction_after_search(case, golden, setup):
    from checkm_b200 import runtime
    from tools import synth
    e = runtime.engine()
    b = synth.make_bin('ws', synth.read_hmms(CPR_HMM), seed=31, n_orfs=400)
    db = e.seqdb(b.residues, b.offsets)
    hits = e.search(runtime.models_for(CPR_HMM), db)
    db.close()
    assert len(hits) > 0
    # the same checks as the reduction's own test (ResultsParser runs on the runtime engine the search above used)
    reduction.test_reduction_matches_reference(case, 'default', golden, setup)
