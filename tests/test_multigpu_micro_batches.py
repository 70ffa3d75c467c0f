"""Gradient accumulation on real GPUs: `tests/mp_micro_batches_worker.py` under torchrun at
every world size the box offers (2 / 4 / 8) must print `ALL OK` — K = 3 micro-batches on the
NVLink fabric against the single-device oracle, P2P and (where available, e.g. at 8) NVLS
buckets, eager and CUDA graph, the joint clip and bf16 master rows.  Skipped on boxes with
fewer GPUs (`multigpu` marker, tests/conftest.py)."""
import os

import pytest

from tests.test_multigpu import _ngpu, _torchrun

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_micro_batches_match_oracle(nproc):
    if _ngpu() < nproc:
        pytest.skip("needs %d GPUs" % nproc)
    r = _torchrun(nproc, os.path.join("tests", "mp_micro_batches_worker.py"), timeout=1000)
    tail = "\n".join((r.stdout + "\n" + r.stderr).splitlines()[-40:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, tail
    assert "FAIL" not in r.stdout, tail
