"""The step's complete host launch plan, pinned.

One eager training step is recorded on the CPU (tests/golden/make_launch_trace.py): every GEMM and
weight-gradient descriptor field by field, every other C-ABI call with its arguments, the stream each
launch goes to, and the data-parallel `grad_ready` signals, with pointers reduced to (buffer, byte offset).
The trace must equal tests/golden/launch_trace.json.gz.  The other CPU plan tests check that the plans
compute the right values; this one notices a launch that moved, changed streams or reads another buffer.

A change that alters the plan on purpose regenerates the fixture with
`python tests/golden/make_launch_trace.py` and says in its description why the plan changed."""
import importlib.util
import json
import os

import pytest

_GEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_launch_trace.py")
_spec = importlib.util.spec_from_file_location("make_launch_trace", _GEN)
gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gen)


@pytest.fixture(scope="module")
def golden():
    return gen.load(gen.FIXTURE)


@pytest.mark.parametrize("case", list(gen.CASES))
def test_launch_trace_matches_the_fixture(golden, case):
    cfg_name, kw = gen.CASES[case]
    # through a JSON round trip, so the comparison sees what the fixture stores
    got = json.loads(json.dumps(gen.record(cfg_name, kw)))
    want = golden[case]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{case}: launch {i} differs\nnow:     {json.dumps(g, sort_keys=True)}\n" \
                       f"fixture: {json.dumps(w, sort_keys=True)}"
    n = min(len(got), len(want))
    assert len(got) == len(want), f"{case}: launch {n} differs ({len(got)} launches, fixture has " \
                                  f"{len(want)})\nnow:     {json.dumps(got[n:n + 1])}\nfixture: {json.dumps(want[n:n + 1])}"
