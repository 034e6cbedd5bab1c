"""The event-graph of the distributed Cholesky (tools/dist_schedule_model.py mirrors the op order of fit_dist_impl):
neither the default order nor the experimental AGP_DIST_SCHED=1 order may deadlock under in-order streams."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
spec = importlib.util.spec_from_file_location("dsm", os.path.join(ROOT, "tools", "dist_schedule_model.py"))
dsm = importlib.util.module_from_spec(spec)
spec.loader.exec_module(dsm)


@pytest.mark.parametrize("R", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("sched2", [False, True])
def test_no_deadlock(R, sched2):
    if R == 1 and sched2:
        pytest.skip("single rank uses cholesky_inplace")
    t = dsm.simulate(dsm.build(8192, R, 512, sched2, 16 if sched2 else 0, 0.7), R)
    assert t > 0
