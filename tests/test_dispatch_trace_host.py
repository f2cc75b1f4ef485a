"""conv_forward's dispatch on CPU: for every case of tests/golden/gen_dispatch_trace.py the float64 emulation of the ops must
record the committed trace (which kernel runs, in what order, with which shapes, plan images and accumulate flags) and the
same emulated outputs (up to last-bit differences of float64 plan building between machines).  Host logic only: the kernels
have their own GPU tests."""
import json

import pytest

from dispatch_emulation import match
from gen_dispatch_trace import CASES, OUT, run_case


@pytest.fixture(scope='module')
def golden():
    with open(OUT) as f:
        return json.load(f)


@pytest.mark.parametrize('name', sorted(CASES))
def test_conv_forward_reproduces_dispatch_trace(golden, name):
    got = json.loads(json.dumps(run_case(name)))           # tuples -> lists, as stored
    want = golden[name]
    assert len(got['trace']) == len(want['trace'])
    for i, (g, w) in enumerate(zip(got['trace'], want['trace'])):
        assert g == w, f'launch {i}'
    assert got['deferred'] == want['deferred'] and len(got['outputs']) == len(want['outputs'])
    for g, w in zip(got['outputs'], want['outputs']):
        assert g.keys() == w.keys() and all(match(g[d], w[d]) for d in w), (g, w)
