"""Run-time switches: the one module that reads the SE3B200_* environment variables.

A switch is on when its variable is set and not empty; numbers are parsed with int() / float().  Every switch selects among
implementations of the same forward (or tunes one); none changes what the model computes beyond rounding.

| variable                    | field             | default          | selects                                                           |
|-----------------------------|-------------------|------------------|-------------------------------------------------------------------|
| SE3B200_NO_LOWRANK          | no_lowrank        | off              | direct K = 128 kernels only, no low-rank radial plan              |
| SE3B200_LOWRANK_MIN_EDGES   | lowrank_min_edges | 16384            | fewest edges of a forward that builds and uses the low-rank plan  |
| SE3B200_LOWRANK_TOL         | lowrank_tol       | ops.LOWRANK_TOL  | residual of the low-rank radial basis, relative to max abs(g)     |
| SE3B200_NO_ALIGNED          | no_aligned        | off              | low-rank path in the global frame (DESIGN.md 4.2-4.3), not 4.4/4.5|
| SE3B200_NO_ZGEMM            | no_zgemm          | off              | R-first edge-aligned kernels (4.4), not one GEMM per (lo, m) (4.5)|
| SE3B200_Z_MODE2             | z_mode2           | off              | four real products per complex one in the m > 0 GEMMs, not three  |
| SE3B200_NO_INPUT_SIDE       | no_input_side     | off              | no input-side contraction (4.3) on the global-frame path          |
| SE3B200_NO_UTABLE           | no_utable         | off              | radial coordinates from the per-edge MLP, not the plan's table    |
| SE3B200_FORCE_SIMT          | force_simt        | off              | fp32 SIMT pairwise kernels and cuBLAS LinearSE3: no tensor cores  |
| SE3B200_NO_LINEAR_TC        | no_linear_tc      | off              | cuBLAS LinearSE3 instead of the tensor-core kernel                |
| SE3B200_NO_ATTN_ROTATE      | no_attn_rotate    | off              | separate rotate-back instead of the one fused into attention      |
| SE3B200_HOST_FRAMES         | host_frames       | off              | edge frames from the float64 torch code of aligned.py             |
| SE3B200_Z_FLUSH             | z_flush           | unset            | tensor-core accumulator drain period in stages (unset: 8; the     |
|                             |                   |                  | m > 0 GEMMs of mode 3 also drain at the end of every weight set)  |
| SE3B200_Z_FLUSH_MULT        | z_flush_mult      | 1                | multiplies the drain period of the ConvSE3 GEMMs                  |
| SE3B200_EDGE_BUDGET_MB      | edge_budget_mb    | unset            | MiB (2^20 bytes) that the edge-level tensors of one ConvSE3 or    |
|                             |                   |                  | attention block may take: its edge work runs over node chunks     |
|                             |                   |                  | sized to fit (model.plan_node_chunks; the result is bit-identical)|
|                             |                   |                  | unset: a quarter of the device's total memory; 0: one-node chunks |
| SE3B200_NO_DECODE_GRAPHS    | no_decode_graphs  | off              | every step of a paged decoder with max_nodes runs eagerly, none   |
|                             |                   |                  | is replayed from a CUDA graph (DESIGN.md 10.3; same rows)         |

The model reads `current()` once per ConvSE3 dispatch, LinearSE3 / AttentionSE3 call, Geometry and pack_weights; ConvSE3
rebuilds its cached dispatch decisions when a switch they depend on changes.  A captured CUDA graph (GraphedForward) replays
the switches it was captured with.  The build-time knobs SE3B200_LIB_TAG, SE3B200_NVCC_DEFS and NVCC belong to build.py.
"""
import contextlib
import dataclasses
import os

from .ops import LOWRANK_TOL


@dataclasses.dataclass(frozen=True)
class Switches:
    no_lowrank: bool = False
    lowrank_min_edges: int = 16384
    lowrank_tol: float = LOWRANK_TOL
    no_aligned: bool = False
    no_zgemm: bool = False
    z_mode2: bool = False
    no_input_side: bool = False
    no_utable: bool = False
    force_simt: bool = False
    no_linear_tc: bool = False
    no_attn_rotate: bool = False
    host_frames: bool = False
    z_flush: int = None
    z_flush_mult: int = 1
    edge_budget_mb: float = None
    no_decode_graphs: bool = False

    def zgemm_flush(self, mode):
        """flush_stages of se3_zgemm_fwd: 0 (the library's default) unless SE3B200_Z_FLUSH or SE3B200_Z_FLUSH_MULT is set."""
        if self.z_flush is None and self.z_flush_mult == 1:
            return 0
        base = self.z_flush if self.z_flush is not None else 8
        return max(1, base * max(1, self.z_flush_mult))

    def linear_flush(self):
        """flush_stages of se3_linear_tc_fwd: 0 (the library's default) unless SE3B200_Z_FLUSH is set."""
        return 0 if self.z_flush is None else max(1, self.z_flush)


FIELDS = tuple(f.name for f in dataclasses.fields(Switches))
ENV = {name: 'SE3B200_' + name.upper() for name in FIELDS}


def current():
    """The switches as the environment sets them now."""
    kw = {}
    for f in dataclasses.fields(Switches):
        v = os.environ.get(ENV[f.name])
        if v:
            kw[f.name] = True if f.type is bool else float(v) if f.type is float else int(v)
    return Switches(**kw)


@contextlib.contextmanager
def override(**fields):
    """Set switches for the duration of the block through their environment variables, so that subprocesses see them too;
    True / a number sets a variable, False / None unsets it.  The previous values come back on exit, also on an exception."""
    unknown = set(fields) - set(FIELDS)
    if unknown:
        raise TypeError(f'unknown switches: {sorted(unknown)}')
    saved = {ENV[name]: os.environ.get(ENV[name]) for name in fields}
    try:
        for name, v in fields.items():
            if v is None or v is False:
                os.environ.pop(ENV[name], None)
            else:
                os.environ[ENV[name]] = '1' if v is True else str(v)
        yield
    finally:
        for var, v in saved.items():
            if v is None:
                os.environ.pop(var, None)
            else:
                os.environ[var] = v
