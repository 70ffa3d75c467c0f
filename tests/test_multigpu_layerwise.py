"""Layer-wise optimizers on real GPUs: `tests/mp_layerwise_worker.py` under torchrun at every
world size the box offers (2 / 4 / 8) must print `ALL OK` — LARS (with and without Nesterov)
and LAMB on the NVLink fabric against the single-device oracle, with and without a clip rule
and micro-batches, eager and CUDA graph, on P2P buckets and, at W >= 4 with NVSwitch
multicast, on NVLS buckets (`dense_nvls=True`).  Skipped on boxes with fewer GPUs
(`multigpu` marker, tests/conftest.py)."""
import os

import pytest

from tests.test_multigpu import _ngpu, _torchrun

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_layerwise_match_oracle(nproc):
    if _ngpu() < nproc:
        pytest.skip("needs %d GPUs" % nproc)
    r = _torchrun(nproc, os.path.join("tests", "mp_layerwise_worker.py"), timeout=1000)
    tail = "\n".join((r.stdout + "\n" + r.stderr).splitlines()[-40:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, tail
    assert "FAIL" not in r.stdout, tail
