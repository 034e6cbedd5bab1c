"""The pipelined multi-GPU schedule (fit_dist_impl, dist_sched == 2) replayed op by op on the CPU: every pair of operations
of one rank that touch the same block column / panel buffer / slice buffer (at least one writing) must be ordered by stream
order or an event edge.  tools/dist_dependency_model.py mirrors the enqueue order of csrc/engine.cu; with the
`split_first` rule switched off it reproduces the race that once surfaced on 8 ranks."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import dist_dependency_model as m  # noqa: E402


@pytest.mark.parametrize("use_oz", [True, False])  # int8-slice path (updates read the slices) / DMMA-FFMA path (they read the panel)
@pytest.mark.parametrize("defer", [True, False])
@pytest.mark.parametrize("R,nto", [(2, 4), (2, 9), (3, 10), (4, 11), (8, 16), (8, 17), (8, 5), (8, 33)])
def test_shipped_schedule_has_no_unordered_conflicts(R, nto, defer, use_oz):
    assert m.check(R, nto, split_first=True, defer=defer, use_oz=use_oz) == []


def test_model_detects_the_round2_race_without_the_first_piece_rule():
    bad = m.check(8, 16, split_first=False)
    assert bad, "the model must see the rest(k-1) / block-column-update(k) conflict"
    assert any(a.startswith("rest") and b.startswith("colupd") and obj[0] == "col" for _, a, b, obj in bad)
