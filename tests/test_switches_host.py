"""The run-time switches (se3_transformer_pytorch_b200/switches.py) on CPU: only the registry reads the environment, every
SE3B200_* name is a registered switch or a build knob, a switch changed between two forwards of the same ConvSE3 takes effect
(under the op emulation of tests/dispatch_emulation.py), and override() restores the environment."""
import glob
import os
import re

import pytest

from dispatch_emulation import Emulation, match
from gen_dispatch_trace import Case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'se3_transformer_pytorch_b200')
BUILD_KNOBS = {'SE3B200_LIB_TAG', 'SE3B200_NVCC_DEFS'}


def _read(path):
    with open(path) as f:
        return f.read()


def _package_sources():
    return [p for p in glob.glob(os.path.join(PKG, '**', '*'), recursive=True) if p.endswith(('.py', '.cu', '.cuh'))]


def test_only_the_registry_reads_the_environment():
    allowed = {os.path.join(PKG, 'switches.py'), os.path.join(PKG, 'build.py')}
    for path in _package_sources() + [os.path.join(ROOT, 'include', 'se3b200.h')]:
        if path not in allowed:
            assert not re.search(r'os\.environ|os\.getenv|getenv\(', _read(path)), path


def test_every_switch_name_is_registered():
    from se3_transformer_pytorch_b200 import switches
    known = set(switches.ENV.values()) | BUILD_KNOBS
    files = _package_sources() + glob.glob(os.path.join(ROOT, '*.md')) + glob.glob(os.path.join(ROOT, 'bench*.py')) + \
        [os.path.join(ROOT, '__graft_entry__.py'), os.path.join(ROOT, 'include', 'se3b200.h')]
    for path in files:
        names = set(re.findall(r'\bSE3B200_[A-Z0-9_]+', _read(path))) - {'SE3B200_H'}      # the header's include guard
        assert names <= known, (path, names - known)


def test_strided_lowrank_entry_point_is_gone():
    from se3_transformer_pytorch_b200 import ops
    assert 'se3_pairwise_lr_strided_fwd' not in _read(os.path.join(ROOT, 'include', 'se3b200.h'))
    assert 'se3_pairwise_lr_strided_fwd' not in ops.EXPORTED_SYMBOLS


def _normalized(trace):
    """The trace without pack_w3 records (direct images depend on the weights alone, so a module keeps them across switch
    changes), with the image labels numbered by first use so that traces of different Emulation objects compare."""
    order = {}

    def norm(v):
        if isinstance(v, list):
            return [norm(u) for u in v]
        m = re.fullmatch(r'(\w+)#\d+(\[.*\])', v) if isinstance(v, str) else None
        return f'{m[1]}#{order.setdefault(v, len(order))}{m[2]}' if m else v

    return [[name, {k: norm(v) for k, v in kw.items()}] for name, kw in trace if name != 'pack_w3']


def _forward(case, emu, **flips):
    n0 = len(emu.trace)
    prints, deferred = case.forward(emu, **flips)
    return _normalized(emu.trace[n0:]), prints, deferred


FLIPS = [
    ('aligned', dict(no_aligned=True)),
    ('zgemm', dict(no_zgemm=True)),
    ('zgemm', dict(z_mode2=True)),
    ('ineligible_pair', dict(no_input_side=True)),
    ('aligned', dict(force_simt=True)),
    ('aligned', dict(no_utable=True)),
    ('aligned', dict(lowrank_tol=1e-8)),
]


@pytest.mark.parametrize('name,flip', FLIPS, ids=[f'{n}-{next(iter(f))}' for n, f in FLIPS])
def test_switch_change_takes_effect_on_the_next_forward(name, flip):
    """A ConvSE3 run once under the defaults and then under `flip` launches exactly what a fresh one launches under `flip`."""
    case, emu = Case(name), Emulation()
    first, _, _ = _forward(case, emu)
    second, prints, deferred = _forward(case, emu, **flip)
    fresh, fresh_prints, fresh_deferred = _forward(Case(name), Emulation(), **flip)
    assert fresh != first, 'the switch does not change this case'
    assert len(second) == len(fresh)
    for i, (g, w) in enumerate(zip(second, fresh)):
        assert g == w, f'launch {i}'
    assert deferred == fresh_deferred
    for g, w in zip(prints, fresh_prints):
        assert g.keys() == w.keys() and all(match(g[d], w[d]) for d in w), (g, w)


def test_released_masters_keep_the_plan_of_pack_weights():
    """With released masters nothing can be rebuilt: the plan of pack_weights stays whatever the switches say, and the direct
    kernels that no_lowrank asks for have no weights left."""
    case, emu = Case('free_master'), Emulation()
    case.forward(emu)                                  # packs the weights, then runs
    first, prints, _ = _forward(case, emu)
    for flip in (dict(no_aligned=True), dict(no_zgemm=True)):
        again, again_prints, _ = _forward(case, emu, **flip)
        assert again == first, flip
        assert all(g.keys() == w.keys() and all(match(g[d], w[d]) for d in w) for g, w in zip(again_prints, prints))
    with pytest.raises(RuntimeError, match='released'):
        case.forward(emu, no_lowrank=True)


def test_override_restores_the_environment_on_an_exception(monkeypatch):
    from se3_transformer_pytorch_b200 import switches
    monkeypatch.setenv('SE3B200_NO_ALIGNED', '1')
    monkeypatch.delenv('SE3B200_FORCE_SIMT', raising=False)
    monkeypatch.setenv('SE3B200_LOWRANK_MIN_EDGES', '7')
    before = switches.current()
    assert before.no_aligned and not before.force_simt and before.lowrank_min_edges == 7
    with pytest.raises(ValueError):
        with switches.override(no_aligned=False, force_simt=True, lowrank_min_edges=None, lowrank_tol=1e-4):
            sw = switches.current()
            assert not sw.no_aligned and sw.force_simt and sw.lowrank_min_edges == 16384 and sw.lowrank_tol == 1e-4
            raise ValueError
    assert os.environ['SE3B200_NO_ALIGNED'] == '1' and 'SE3B200_FORCE_SIMT' not in os.environ
    assert os.environ['SE3B200_LOWRANK_MIN_EDGES'] == '7' and switches.current() == before
    with pytest.raises(TypeError):
        with switches.override(no_such_switch=True):
            pass
