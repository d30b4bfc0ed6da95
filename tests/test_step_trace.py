"""CPU: the samplers' region-blend kernel calls (entry point, scalars, which buffer goes where, noise draws) against the
trace recorded by tests/gen_step_trace.py, for every scheduler, both samplers and the fused peer-exchange path."""
import json

import pytest

from tests import gen_step_trace as gst

_GOLDEN = json.load(open(gst.GOLDEN))
_CASES = gst.cases()


def test_golden_covers_every_case():
    assert set(_GOLDEN) == set(_CASES)


@pytest.mark.parametrize("name", sorted(_CASES))
def test_step_trace(name):
    got = json.loads(json.dumps(_CASES[name]()))   # tuples -> lists, as stored
    want = _GOLDEN[name]
    for k, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: event {k} differs\n got  {g}\n want {w}"
    assert len(got) == len(want), f"{name}: {len(got)} events, the golden has {len(want)}"
