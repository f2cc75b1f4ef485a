"""ctypes binding of libse3b200.so (C ABI in include/se3b200.h) for torch CUDA tensors.

PyTorch is plumbing here: it owns device memory and the current stream; every op below hands raw device pointers
and the stream handle to the hand-written sm_90a kernels.  There is NO CPU fallback: calling an op with a
non-CUDA tensor, or without the compiled library, raises.
"""
import ctypes
import os
import threading
from typing import NamedTuple

import numpy as np
import torch

from . import build as _build

_PKG = os.path.dirname(os.path.abspath(__file__))
_lib = None
_lock = threading.Lock()

c_void_p, c_int, c_int64, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float

_SIGNATURES = {
    'se3_last_error': (ctypes.c_char_p, []),
    'se3_abi_version': (c_int, []),
    'se3_knn_fwd': (c_int, [c_void_p] * 7 + [c_int, c_int64, c_int, c_float, c_int] + [c_void_p] * 4 + [c_void_p]),
    'se3_knn_rows_fwd': (c_int, [c_void_p] * 3 + [c_int, c_int64, c_int64, c_int, c_int, c_int, c_float, c_int] + [c_void_p] * 5),
    'se3_knn_rows_packed_fwd': (c_int, [c_void_p] * 7 + [c_int, c_int64, c_int64, c_int, c_int, c_float, c_int] + [c_void_p] * 5),
    'se3_knn_rows_paged_fwd': (c_int, [c_void_p] * 8 + [c_int, c_int64, c_int, c_int, c_int, c_float, c_int] + [c_void_p] * 6),
    'se3_decode_plan_fwd': (c_int, [c_void_p, c_int, c_int, c_int, c_int64, c_void_p, c_void_p]),
    'se3_knn_rows_paged_bucket_fwd': (c_int, [c_void_p] * 3 + [c_int] * 5 + [c_float, c_int] + [c_void_p] * 6),
    'se3_prefix_keys_fwd': (c_int, [c_void_p, c_int64, c_int64] + [c_void_p] * 3 + [c_int] + [c_void_p] * 4 + [c_int, c_void_p, c_void_p]),
    'se3_pair_lookup_fwd': (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    'se3_gather_pairs_fwd': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    'se3_basis_fwd': (c_int, [c_void_p, c_int64, c_int] + [c_void_p] * 5 + [c_int, c_void_p, c_void_p]),
    'se3_radial_trunk_fwd': (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    'se3_tbuild_fwd': (c_int, [c_void_p] * 3 + [c_int] * 7 + [c_int64, c_int64, c_void_p, c_void_p]),
    'se3_pairwise_simt_fwd': (c_int, [c_void_p] * 4 + [c_int64] + [c_int] * 5 + [c_void_p, c_void_p]),
    'se3_w3_image_bytes': (c_int64, [c_int, c_int, c_int]),
    'se3_pack_w3': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    'se3_pairwise_tc_fwd': (c_int, [c_void_p] * 3 + [c_int64] + [c_int] * 5 + [c_void_p, c_void_p]),
    'se3_pairwise_tc_debug': (c_int, [c_void_p] * 3 + [c_int64] + [c_int] * 5 + [c_void_p, c_void_p, c_void_p]),
    'se3_lowrank_image_bytes': (c_int64, [c_int, c_int, c_int, c_int]),
    'se3_pack_lowrank': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    'se3_pairwise_lr_fwd': (c_int, [c_void_p] * 3 + [c_int64] + [c_int] * 6 + [c_void_p, c_void_p]),
    'se3_fold_basis_fwd': (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    'se3_fold_basis_cm_fwd': (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    'se3_rotate_back_fwd': (c_int, [c_void_p] * 5 + [c_int64, c_int, c_int, c_void_p, c_void_p]),
    'se3_radial_trunk_u_fwd': (c_int, [c_void_p, c_int64, c_int, c_int] + [c_void_p] * 8),
    'se3_radial_table_fwd': (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int, c_float, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    'se3_frames_fwd': (c_int, [c_void_p, c_int64, c_int] + [c_void_p] * 5),
    'se3_rotgather_fwd': (c_int, [c_void_p] * 3 + [c_int] * 5 + [c_int64, c_int64, c_void_p, c_void_p]),
    'se3_rotate_pool_fwd': (c_int, [c_void_p] * 4 + [c_int64, c_int, c_int, c_int, c_void_p, c_void_p]),
    'se3_linear_tc_fwd': (c_int, [c_void_p] * 4 + [c_int64, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    'se3_pow2_scale_fwd': (c_int, [c_void_p, c_int64, c_int, c_void_p, c_void_p]),
    'se3_rowabsmax_fwd': (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p]),
    'se3_edge_scale_fwd': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    'se3_zgemm_tile_n': (c_int, [c_int, c_int]),
    'se3_zgemm_image_bytes': (c_int64, [c_int, c_int, c_int]),
    'se3_zgemm_pack': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    'se3_zgemm_fwd': (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_int64, c_int, c_int, c_int, c_void_p]),
    'se3_zgemm_split_units': (c_int, [c_void_p, c_int, c_int, c_int, c_int]),
    'se3_zgemm_workspace_bytes': (c_int64, [c_void_p, c_int, c_int64, c_int, c_int, c_int]),
    'se3_zgemm_split_fwd': (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_int64, c_int, c_int, c_int,
                                    c_int, c_void_p, c_int64, c_void_p]),
    'se3_pool_fwd': (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int64, c_void_p, c_void_p]),
    'se3_norm_fwd': (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_float, c_int, c_void_p, c_void_p]),
    'se3_attn_aligned_fwd': (c_int, [c_void_p] * 4 + [c_int] + [c_void_p] * 7 + [c_int, c_void_p] + [c_int] * 7 + [c_float, c_void_p, c_void_p]),
    'se3_attn_fwd': (c_int, [c_void_p] * 10 + [c_int, c_void_p] + [c_int] * 7 + [c_float, c_void_p, c_void_p]),
}
EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def lib():
    """Load (building if the sources changed) libse3b200.so.  Raises if it cannot be built/loaded."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                path = _build.build()
                handle = ctypes.CDLL(path)
                for name, (res, args) in _SIGNATURES.items():
                    fn = getattr(handle, name)       # AttributeError if the symbol is missing -> loud failure
                    fn.restype = res
                    fn.argtypes = args
                _lib = handle
    return _lib


LAUNCHES = 0          # number of libse3b200 kernel launches issued by this process (bench.py reports it)
PROFILE = None        # when a list: every launch appends (kernel, start_event, end_event, reference-formulation FLOPs,
                      # algorithmic (unpadded) bytes, tag, issued tensor-core FLOPs (every pass counted), issued fp32 FMA FLOPs)


def _check(rc):
    global LAUNCHES
    if rc != 0:
        raise RuntimeError('libse3b200: ' + lib().se3_last_error().decode())
    LAUNCHES += 1


class _timed:
    """CUDA-event bracket on the launching stream around one kernel launch (only when PROFILE is enabled)."""

    def __init__(self, name, flops=0, nbytes=0, tag='', mma=0, fma=0):
        self.name, self.flops, self.nbytes, self.tag, self.mma, self.fma = name, flops, nbytes, tag, mma, fma

    def __enter__(self):
        if PROFILE is not None:
            self.start = torch.cuda.Event(enable_timing=True)
            self.end = torch.cuda.Event(enable_timing=True)
            self.start.record()
        return self

    def __exit__(self, *exc):
        if PROFILE is not None and exc[0] is None:
            self.end.record()
            PROFILE.append((self.name, self.start, self.end, self.flops, self.nbytes, self.tag, self.mma, self.fma))
        return False


def _require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError('se3_transformer_pytorch_b200 runs on CUDA (sm_90a) only: got a tensor on %s; '
                               'there is no CPU path' % t.device)


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _f32(t):
    if t.dtype != torch.float32:
        raise RuntimeError(f'se3_transformer_pytorch_b200 computes in float32 (got {t.dtype})')
    return t.contiguous()


def _u8(t):
    return None if t is None else t.contiguous().view(torch.uint8) if t.dtype == torch.bool else t.contiguous().to(torch.uint8)


# ---------------------------------------------------------------------------------------------------------
# K1
# ---------------------------------------------------------------------------------------------------------
class PairRows(NamedTuple):
    """A sparse pair input as sorted column lists (se3_pairs of se3_knn_fwd): row r = b * n + i (or i when shared) holds
    entries ptr[r] .. ptr[r+1] of cols (ascending, unique) and values."""
    ptr: torch.Tensor         # int64 [rows + 1]
    cols: torch.Tensor        # int32 [nnz], node index inside the cloud
    values: torch.Tensor      # [nnz, ...] in the input's dtype
    shared: bool              # one [n, n] list for every cloud of the batch (batch stride 0)


def pair_rows(rows, cols, values, num_rows, shared):
    """PairRows from entries sorted by (row, col): rows int64 [nnz] in [0, num_rows), cols [nnz]."""
    ptr = torch.zeros(num_rows + 1, dtype=torch.int64, device=rows.device)
    ptr[1:] = torch.bincount(rows, minlength=num_rows).cumsum(0)
    return PairRows(ptr, cols.to(torch.int32), values, shared)


def coo_to_rows(t, n):
    """A torch.sparse_coo pair input [n, n] or [B, n, n] (sparse dims; dense dims after them stay in the values) -> PairRows.
    Coalescing sums duplicate entries, as to_dense() does; stored zeros and diagonal entries are kept.  [n, n] and [1, n, n]
    give one shared list.  Torch only, so it also runs on the CPU."""
    t = t.coalesce()
    ind = t.indices()
    if t.sparse_dim() == 2:
        rows, cols, B = ind[0], ind[1], 1
    else:
        rows, cols, B = ind[0] * n + ind[1], ind[2], t.shape[0]
    return pair_rows(rows, cols, t.values(), B * n, B == 1)


def _row_args(rows, b, n):
    """(ptr, cols, nnz, batch stride) of a PairRows for a batch [b, n]; an empty list keeps a non-NULL column pointer, since
    NULL means no list."""
    want = (n if rows.shared else b * n) + 1
    if rows.ptr.dtype != torch.int64 or rows.ptr.shape != (want,) or rows.cols.dtype != torch.int32 or rows.cols.dim() != 1:
        raise ValueError(f'pair rows for b, n = {(b, n)} need int64 row pointers [{want}] and int32 columns [nnz], got '
                         f'{rows.ptr.dtype} {tuple(rows.ptr.shape)} and {rows.cols.dtype} {tuple(rows.cols.shape)}')
    cols = rows.cols.contiguous() if rows.cols.numel() else torch.zeros(1, dtype=torch.int32, device=rows.cols.device)
    return rows.ptr.contiguous(), cols, rows.cols.numel(), 0 if rows.shared else n


def pair_lookup(rows, idx):
    """Position of every neighbour idx [b, n, k] in the PairRows rows (int64 [b, n, k]), -1 where its row lacks the pair:
    rows.values indexed with a zero row appended for -1 are the pair values on the neighbour list."""
    _require_cuda(idx, rows.ptr, rows.cols)
    b, n, k = idx.shape
    ptr, cols, nnz, stride = _row_args(rows, b, n)
    out = torch.empty((b, n, k), dtype=torch.int64, device=idx.device)
    with torch.cuda.device(idx.device), _timed('pair_lookup', nbytes=16 * b * n * k):
        _check(lib().se3_pair_lookup_fwd(_p(ptr), _p(cols), nnz, stride, _p(idx.contiguous()), b, n, k, _p(out), _stream()))
    return out


MAX_CLOUD = 4097      # nodes per cloud of the shared-memory sort (n - 1 <= 4096 columns)
KNN_MAX_K = 4096      # neighbours per node: the longest list the tiled search keeps next to its tile


def pair_offsets(seqlens):
    """Start of each cloud's [n_c, n_c] block in a flattened packed pair input: sum of n_c'^2 over the clouds before it."""
    off = [0]
    for n in seqlens[:-1]:
        off.append(off[-1] + n * n)
    return off


class _Pairs(ctypes.Structure):
    _fields_ = [('dense', c_void_p), ('row_ptr', c_void_p), ('cols', c_void_p), ('nnz', c_int64), ('shared', c_int)]


def knn(coors, k, valid_radius, *, node_mask=None, neighbor_mask=None, sparse_adj=None, causal=False, seqlens=None, K=None):
    """Neighbour graph (reference se3_transformer_pytorch.py:1171-1294) of a padded or a packed batch.
    Padded: coors [b, n, 3], k neighbours of every node, node_mask [b, n].  Returns idx int64 [b, n, k] (indices inside the
    cloud), mask bool [b, n, k], rel_pos [b, n, k, 3], rel_dist [b, n, k].
    Packed (SE3Transformer.forward_packed): clouds of seqlens[c] nodes laid end to end in coors [T, 3], each searched on its
    own for k[c] neighbours, K >= max k_c slots per node (default max k_c; slots past k_c repeat slot k_c - 1, masked).
    Returns idx int64 [T, K] (global node indices), mask bool [T, K], rel_pos [T, K, 3], rel_dist [T, K].
    neighbor_mask / sparse_adj: a tensor ([n, n], [1, n, n] or [b, n, n] padded; the clouds' [n_c, n_c] matrices flattened end
    to end when packed) or, padded only, a PairRows; the two give the same results bit for bit."""
    pair_inputs = [t for t in (neighbor_mask, sparse_adj) if t is not None]
    _require_cuda(coors, node_mask, *(x for t in pair_inputs for x in (t[:2] if isinstance(t, PairRows) else (t,))))
    coors = _f32(coors)
    dev = coors.device
    cu = kc = off = None
    if seqlens is None:
        b, n, _ = coors.shape
        T, K = b * n, k
        if node_mask is not None and node_mask.shape != (b, n):
            raise ValueError(f'knn: node_mask must be [b, n] = {(b, n)}, got {tuple(node_mask.shape)}')
    else:
        seqlens, k = [int(v) for v in seqlens], [int(v) for v in k]
        b, T = len(seqlens), sum(seqlens)
        n = T                                       # se3_knn_fwd takes the number of all nodes here
        if b == 0 or coors.shape != (T, 3):
            raise ValueError(f'knn: coors must be [sum(seqlens), 3] = {(T, 3)} for {b} clouds, got {tuple(coors.shape)}')
        if len(k) != b:
            raise ValueError(f'knn: k has {len(k)} entries for {b} clouds')
        if min(seqlens) < 2 or max(seqlens) > MAX_CLOUD:
            raise ValueError(f'knn: every cloud needs 2 .. {MAX_CLOUD} nodes, got lengths {min(seqlens)} .. {max(seqlens)}')
        K = max(k) if K is None else K
        if any(not 1 <= k_c <= n_c - 1 for k_c, n_c in zip(k, seqlens)) or K < max(k):
            raise ValueError(f'knn: need 1 <= k_c <= n_c - 1 and K >= max k_c (K = {K}, k = {k}, n = {seqlens})')
        cu = torch.tensor([0] + seqlens, dtype=torch.int64).cumsum(0).to(dev)
        kc = torch.tensor(k, dtype=torch.int32).to(dev)
        if any(torch.is_tensor(t) for t in pair_inputs):
            off = torch.tensor(pair_offsets(seqlens), dtype=torch.int64).to(dev)
    nm = _u8(node_mask)
    keep, args, nbytes = [], [], 12 * T + 25 * T * K + (0 if nm is None else nm.numel())
    for name, t in (('neighbor_mask', neighbor_mask), ('sparse_adj', sparse_adj)):
        if t is None:
            args.append(None)
            continue
        if isinstance(t, PairRows):
            ptr, cols, nnz, stride = _row_args(t, T // n, n)   # (packed clouds refuse column lists)
            keep += [ptr, cols]
            args.append(ctypes.byref(_Pairs(None, _p(ptr), _p(cols), nnz, int(stride == 0))))
            nbytes += 4 * nnz
            continue
        if seqlens is not None:
            npairs = sum(n_c * n_c for n_c in seqlens)
            if t.shape != (npairs,):
                raise ValueError(f'knn: {name} must be the flattened per-cloud [n_c, n_c] matrices, [{npairs}], got {tuple(t.shape)}')
        elif t.shape[-2:] != (n, n) or t.dim() not in (2, 3) or (t.dim() == 3 and t.shape[0] not in (1, b)):
            raise ValueError(f'knn: {name} must be [n, n], [1, n, n] or [b, n, n] with b, n = {(b, n)}, got {tuple(t.shape)}')
        t = _u8(t)
        keep.append(t)
        args.append(ctypes.byref(_Pairs(_p(t), None, None, 0, int(seqlens is None and (t.dim() == 2 or t.shape[0] == 1)))))
        nbytes += t.numel()
    rows = (T, K) if seqlens is not None else (b, n, K)
    idx = torch.empty(rows, dtype=torch.int64, device=dev)
    mask = torch.empty(rows, dtype=torch.uint8, device=dev)
    rel_pos = torch.empty((*rows, 3), dtype=torch.float32, device=dev)
    rel_dist = torch.empty(rows, dtype=torch.float32, device=dev)
    valid_radius = float(min(valid_radius, 3.0e38))
    with torch.cuda.device(dev), _timed('knn' if seqlens is None else 'knn_varlen', nbytes=nbytes):
        _check(lib().se3_knn_fwd(_p(coors), _p(cu), _p(kc), _p(off), _p(nm), *args, b, n, K, valid_radius, int(bool(causal)),
                                 _p(idx), _p(mask), _p(rel_pos), _p(rel_dist), _stream()))
    return idx, mask.view(torch.bool), rel_pos, rel_dist


def knn_rows(coors, n, row0, m, k, valid_radius, *, node_mask=None, neighbor_mask=None, causal=False):
    """The neighbour search of rows row0 .. row0 + m of clouds stored with room to grow: coors [b, ld, 3] and node_mask [b, ld]
    (contiguous, ld >= n) hold b clouds of which the first n nodes are searched; neighbor_mask [b, m, n] holds the new rows'
    masks.  Returns idx int64 [b, m, k] (local indices), mask bool [b, m, k], rel_pos [b, m, k, 3], rel_dist [b, m, k]: the rows
    of knn() over the same b clouds of n nodes, bit for bit."""
    _require_cuda(coors, node_mask, neighbor_mask)
    if coors.dtype != torch.float32 or not coors.is_contiguous() or coors.dim() != 3:
        raise ValueError('knn_rows: coors must be a contiguous float32 [b, ld, 3] tensor')
    b, ld, _ = coors.shape
    if node_mask is not None and (node_mask.shape != (b, ld) or not node_mask.is_contiguous()):
        raise ValueError(f'knn_rows: node_mask must be a contiguous [b, ld] = {(b, ld)} tensor, got {tuple(node_mask.shape)}')
    if neighbor_mask is not None and neighbor_mask.shape != (b, m, n):
        raise ValueError(f'knn_rows: neighbor_mask must be [b, m, n] = {(b, m, n)}, got {tuple(neighbor_mask.shape)}')
    dev = coors.device
    idx = torch.empty((b, m, k), dtype=torch.int64, device=dev)
    mask = torch.empty((b, m, k), dtype=torch.uint8, device=dev)
    rel_pos = torch.empty((b, m, k, 3), dtype=torch.float32, device=dev)
    rel_dist = torch.empty((b, m, k), dtype=torch.float32, device=dev)
    nm, nbr = _u8(node_mask), _u8(neighbor_mask)
    with torch.cuda.device(dev), _timed('knn_rows', nbytes=12 * b * n + 25 * b * m * k):
        _check(lib().se3_knn_rows_fwd(_p(coors), _p(nm), _p(nbr), b, n, ld, row0, m, k, float(min(valid_radius, 3.0e38)),
                                      int(bool(causal)), _p(idx), _p(mask), _p(rel_pos), _p(rel_dist), _stream()))
    return idx, mask.view(torch.bool), rel_pos, rel_dist


def knn_rows_packed(coors, slots, n_prev, seqlens, k, valid_radius, *, neighbor_mask=None, causal=False):
    """The neighbour search of the new rows of clouds of different lengths that grow on their own (PackedCausalDecoder): coors
    [S, ld, 3] (contiguous float32) holds cloud c in row slots[c]; its seqlens[c] >= 1 new rows are nodes n_prev[c] + r,
    searched over its first n_cur_c = n_prev[c] + seqlens[c] nodes for k[c] neighbours.  neighbor_mask: None, or a list with
    one [seqlens[c], n_cur_c] bool mask (or None) per cloud.  Returns idx int64 [M, K] (M = sum(seqlens), K = max k_c; indices
    slots[c] * ld + j in the [S * ld] view), mask bool [M, K], rel_pos [M, K, 3], rel_dist [M, K]: cloud c's rows are those of
    knn_rows on that cloud alone in slots < k_c, and slots >= k_c repeat slot k_c - 1, masked.  The per-cloud descriptors are
    checked here and uploaded in one copy; nothing is read back."""
    if coors.dtype != torch.float32 or not coors.is_contiguous() or coors.dim() != 3 or coors.shape[2] != 3:
        raise ValueError('knn_rows_packed: coors must be a contiguous float32 [S, ld, 3] tensor')
    masks = list(neighbor_mask) if neighbor_mask is not None else None
    _require_cuda(coors, *(masks or ()))
    S, ld, _ = coors.shape
    slots, n_prev, seqlens, k = ([int(v) for v in a] for a in (slots, n_prev, seqlens, k))
    B = len(slots)
    if B == 0 or not len(n_prev) == len(seqlens) == len(k) == B:
        raise ValueError(f'knn_rows_packed: slots, n_prev, seqlens and k need one entry per cloud, got lengths '
                         f'{[len(slots), len(n_prev), len(seqlens), len(k)]}')
    n_cur = [p + m for p, m in zip(n_prev, seqlens)]
    for c in range(B):
        if not (0 <= slots[c] < S and n_prev[c] >= 0 and seqlens[c] >= 1 and 2 <= n_cur[c] <= ld and 1 <= k[c] <= n_cur[c] - 1):
            raise ValueError(f'knn_rows_packed: cloud {c} needs 0 <= slot < {S}, n_prev >= 0, m >= 1, 2 <= n_prev + m <= ld = {ld} '
                             f'and 1 <= k <= n_prev + m - 1 (got slot={slots[c]} n_prev={n_prev[c]} m={seqlens[c]} k={k[c]})')
    K, M = max(k), sum(seqlens)
    if K > KNN_MAX_K:
        raise ValueError(f'knn_rows_packed: {K} neighbours exceed {KNN_MAX_K}, the longest list the tiled search keeps')
    if M >= 2 ** 31:
        raise ValueError(f'knn_rows_packed: {M} rows exceed the 1-D grid')
    off, nbr = _row_masks('knn_rows_packed', masks, seqlens, n_cur)
    cu = [0]
    for m in seqlens:
        cu.append(cu[-1] + m)
    dev = coors.device
    desc = torch.tensor(cu + slots + n_prev + k + off, dtype=torch.int64).to(dev)      # the one upload of the step's descriptors
    cu_d, slot_d, prev_d, k_d, off_d = desc[:B + 1], desc[B + 1:2 * B + 1], desc[2 * B + 1:3 * B + 1], desc[3 * B + 1:4 * B + 1], desc[4 * B + 1:]
    idx = torch.empty((M, K), dtype=torch.int64, device=dev)
    mask = torch.empty((M, K), dtype=torch.uint8, device=dev)
    rel_pos = torch.empty((M, K, 3), dtype=torch.float32, device=dev)
    rel_dist = torch.empty((M, K), dtype=torch.float32, device=dev)
    nbytes = 12 * sum(n_cur) + 25 * M * K + (0 if nbr is None else nbr.numel())
    with torch.cuda.device(dev), _timed('knn_rows_packed', nbytes=nbytes):
        _check(lib().se3_knn_rows_packed_fwd(_p(coors), _p(nbr), _p(cu_d), _p(slot_d), _p(prev_d), _p(k_d), _p(off_d), B, M, ld,
                                             max(n_cur), K, float(min(valid_radius, 3.0e38)), int(bool(causal)), _p(idx), _p(mask),
                                             _p(rel_pos), _p(rel_dist), _stream()))
    return idx, mask.view(torch.bool), rel_pos, rel_dist


def _row_masks(api, masks, seqlens, n_cur):
    """The new rows' neighbour masks of a ragged row search (None, or one [m_c, n_cur_c] bool mask or None per cloud) end to end
    as uint8: (per-cloud offsets, -1 for none, and the buffer or None)."""
    B = len(seqlens)
    off, nbr = [-1] * B, None
    if masks is not None:
        if len(masks) != B:
            raise ValueError(f'{api}: neighbor_mask must have one entry per cloud ({B}), got {len(masks)}')
        parts, at = [], 0
        for c, t in enumerate(masks):
            if t is None:
                continue
            if tuple(t.shape) != (seqlens[c], n_cur[c]):
                raise ValueError(f'{api}: neighbor_mask[{c}] must be [m, n_cur] = {(seqlens[c], n_cur[c])}, got {tuple(t.shape)}')
            off[c] = at
            at += t.numel()
            parts.append(_u8(t).reshape(-1))
        nbr = torch.cat(parts) if parts else None
    return off, nbr


def knn_rows_paged(pool, tables, n_prev, seqlens, k, valid_radius, *, neighbor_mask=None, causal=False):
    """The neighbour search of the new rows of clouds kept in pages (PagedCausalDecoder): pool [pages, P, 3] (contiguous float32)
    holds node j of cloud c at row tables[c][j // P] * P + j % P of its [pages * P, 3] view; tables[c] lists at least
    ceil(n_cur_c / P) page ids.  n_prev, seqlens, k and neighbor_mask are as in knn_rows_packed.  Returns idx int64 [M, K] (the
    neighbours' pool rows), col int64 [M, K] (their columns j in the cloud), mask bool [M, K], rel_pos [M, K, 3] and rel_dist
    [M, K]: cloud c's rows are knn_rows_packed's for the same cloud stored contiguously, with col its local indices.  The
    descriptors and page lists are checked here and uploaded in one copy; nothing is read back."""
    if pool.dtype != torch.float32 or not pool.is_contiguous() or pool.dim() != 3 or pool.shape[2] != 3:
        raise ValueError('knn_rows_paged: pool must be a contiguous float32 [pages, page_size, 3] tensor')
    masks = list(neighbor_mask) if neighbor_mask is not None else None
    _require_cuda(pool, *(masks or ()))
    pages, P, _ = pool.shape
    tables = [[int(v) for v in t] for t in tables]
    n_prev, seqlens, k = ([int(v) for v in a] for a in (n_prev, seqlens, k))
    B = len(tables)
    if B == 0 or not len(n_prev) == len(seqlens) == len(k) == B:
        raise ValueError(f'knn_rows_paged: tables, n_prev, seqlens and k need one entry per cloud, got lengths '
                         f'{[len(tables), len(n_prev), len(seqlens), len(k)]}')
    n_cur = [p + m for p, m in zip(n_prev, seqlens)]
    for c in range(B):
        if not (n_prev[c] >= 0 and seqlens[c] >= 1 and 2 <= n_cur[c] < 2 ** 31 and 1 <= k[c] <= n_cur[c] - 1):
            raise ValueError(f'knn_rows_paged: cloud {c} needs n_prev >= 0, m >= 1, 2 <= n_prev + m < 2^31 and '
                             f'1 <= k <= n_prev + m - 1 (got n_prev={n_prev[c]} m={seqlens[c]} k={k[c]})')
        need = -(-n_cur[c] // P)
        if len(tables[c]) < need or not all(0 <= p < pages for p in tables[c][:need]):
            raise ValueError(f'knn_rows_paged: cloud {c} needs {need} page ids in [0, {pages}) for its {n_cur[c]} nodes, got '
                             f'{tables[c][:need]}')
    K, M = max(k), sum(seqlens)
    if K > KNN_MAX_K:
        raise ValueError(f'knn_rows_paged: {K} neighbours exceed {KNN_MAX_K}, the longest list the tiled search keeps')
    if M >= 2 ** 31:
        raise ValueError(f'knn_rows_paged: {M} rows exceed the 1-D grid')
    off, nbr = _row_masks('knn_rows_paged', masks, seqlens, n_cur)
    cu, toff = [0], [0]
    for m, t in zip(seqlens, tables):
        cu.append(cu[-1] + m)
        toff.append(toff[-1] + len(t))
    if toff[-1] >= 2 ** 31:
        raise ValueError(f'knn_rows_paged: {toff[-1]} page ids exceed 2^31')
    # the one upload of the step: int64 descriptors [cu_rows | n_prev | k | pair_off | table_off], then the int32 page ids
    nd = 5 * B + 1
    host = torch.empty(2 * nd + toff[-1], dtype=torch.int32)
    host[:2 * nd].view(torch.int64).copy_(torch.tensor(cu + n_prev + k + off + toff[:-1], dtype=torch.int64))
    host[2 * nd:] = torch.tensor([p for t in tables for p in t], dtype=torch.int32)
    dev = pool.device
    buf = host.to(dev)
    desc, page_ids = buf[:2 * nd].view(torch.int64), buf[2 * nd:]
    cu_d, prev_d, k_d, off_d, toff_d = desc[:B + 1], desc[B + 1:2 * B + 1], desc[2 * B + 1:3 * B + 1], desc[3 * B + 1:4 * B + 1], desc[4 * B + 1:]
    idx = torch.empty((M, K), dtype=torch.int64, device=dev)
    col = torch.empty((M, K), dtype=torch.int64, device=dev)
    mask = torch.empty((M, K), dtype=torch.uint8, device=dev)
    rel_pos = torch.empty((M, K, 3), dtype=torch.float32, device=dev)
    rel_dist = torch.empty((M, K), dtype=torch.float32, device=dev)
    nbytes = 16 * sum(n_cur) + 33 * M * K + (0 if nbr is None else nbr.numel())
    with torch.cuda.device(dev), _timed('knn_rows_paged', nbytes=nbytes):
        _check(lib().se3_knn_rows_paged_fwd(_p(pool), _p(page_ids), _p(nbr), _p(cu_d), _p(prev_d), _p(k_d), _p(off_d), _p(toff_d),
                                            B, M, P, max(n_cur), K, float(min(valid_radius, 3.0e38)), int(bool(causal)), _p(idx),
                                            _p(col), _p(mask), _p(rel_pos), _p(rel_dist), _stream()))
    return idx, col, mask.view(torch.bool), rel_pos, rel_dist


def decode_desc_words(num_clouds, page_ids):
    """int32 words of the descriptor of a padded paged decoding step (se3b200.h, se3_decode_plan_fwd) for num_clouds clouds
    and room for page_ids page ids, rounded up to whole int64 words."""
    return 2 * (5 * num_clouds + 1) + page_ids + page_ids % 2


def fill_decode_desc(buf, num_clouds, n_prev, seqlens, k, tables):
    """Write the descriptor of a step that appends seqlens[c] nodes to cloud c of n_prev[c] nodes with k[c] neighbours into the
    int32 host tensor buf (decode_desc_words long): cu_rows, n_prev, k, pair_off and table_off for num_clouds clouds, those past
    the step's empty, then the page ids of tables[c] (the ones the step reads, in node order).  Returns the step's rows M."""
    B, nd = len(seqlens), 5 * num_clouds + 1
    if not 1 <= B <= num_clouds or not len(n_prev) == len(k) == len(tables) == B:
        raise ValueError(f'fill_decode_desc: need 1 <= {B} clouds <= num_clouds = {num_clouds}, one n_prev, k and table each')
    words = buf.numpy()
    head = words[:2 * nd].view(np.int64)
    m = np.asarray(seqlens, dtype=np.int64)
    n_cur = np.asarray(n_prev, dtype=np.int64) + m
    lens = np.fromiter((len(t) for t in tables), dtype=np.int64, count=B)
    if 2 * nd + int(lens.sum()) > words.shape[0]:
        raise ValueError(f'fill_decode_desc: {int(lens.sum())} page ids exceed the descriptor\'s room of {words.shape[0] - 2 * nd}')
    head[:] = 0
    head[1:B + 1] = np.cumsum(m)
    head[B + 1:num_clouds + 1] = head[B]
    head[num_clouds + 1:num_clouds + 1 + B] = n_prev
    head[2 * num_clouds + 1:3 * num_clouds + 1] = 1
    head[2 * num_clouds + 1:2 * num_clouds + 1 + B] = k
    head[3 * num_clouds + 2:3 * num_clouds + 1 + B] = np.cumsum(m * n_cur)[:-1]
    head[4 * num_clouds + 2:4 * num_clouds + 1 + B] = np.cumsum(lens)[:-1]
    words[2 * nd:2 * nd + int(lens.sum())] = [p for t in tables for p in t]
    return int(head[B])


def decode_plan(desc, num_clouds, rows, page_size, scratch_row):
    """Per row of a paged decoding step padded to `rows` rows, from its device descriptor (fill_decode_desc): int64 [4, rows] of
    the node's position in its cloud, its pool row, where its pair row starts in the step's concatenated pair inputs, and its
    cloud.  Padding rows repeat the last row, except for their pool rows scratch_row, scratch_row + 1, ..."""
    _require_cuda(desc)
    out = torch.empty((4, rows), dtype=torch.int64, device=desc.device)
    with torch.cuda.device(desc.device), _timed('decode_plan', nbytes=64 * rows):
        _check(lib().se3_decode_plan_fwd(_p(desc), num_clouds, rows, page_size, scratch_row, _p(out), _stream()))
    return out


def knn_rows_paged_bucket(pool, desc, num_clouds, rows, n_max, K, valid_radius, *, neighbor_mask=None, causal=False):
    """knn_rows_paged of a step padded to `rows` rows, described by its device descriptor (fill_decode_desc) instead of host
    lists: every cloud has k = K; neighbor_mask: None or the step's masks concatenated as bytes at the descriptor's pair_off.
    n_max bounds every cloud's length.  Padding rows repeat the last row's search.  Nothing is read back."""
    _require_cuda(pool, desc, neighbor_mask)
    if pool.dtype != torch.float32 or not pool.is_contiguous() or pool.dim() != 3 or pool.shape[2] != 3:
        raise ValueError('knn_rows_paged_bucket: pool must be a contiguous float32 [pages, page_size, 3] tensor')
    if K > KNN_MAX_K:
        raise ValueError(f'knn_rows_paged_bucket: {K} neighbours exceed {KNN_MAX_K}, the longest list the tiled search keeps')
    dev = pool.device
    idx = torch.empty((rows, K), dtype=torch.int64, device=dev)
    col = torch.empty((rows, K), dtype=torch.int64, device=dev)
    mask = torch.empty((rows, K), dtype=torch.uint8, device=dev)
    rel_pos = torch.empty((rows, K, 3), dtype=torch.float32, device=dev)
    rel_dist = torch.empty((rows, K), dtype=torch.float32, device=dev)
    nbr = _u8(neighbor_mask)
    with torch.cuda.device(dev), _timed('knn_rows_paged', nbytes=33 * rows * K):
        _check(lib().se3_knn_rows_paged_bucket_fwd(_p(pool), _p(desc), _p(nbr), num_clouds, rows, pool.shape[1], n_max, K,
                                                   float(min(valid_radius, 3.0e38)), int(bool(causal)), _p(idx), _p(col), _p(mask),
                                                   _p(rel_pos), _p(rel_dist), _stream()))
    return idx, col, mask.view(torch.bool), rel_pos, rel_dist


def prefix_keys(feats, coors, seqlens, n_prev=None, *, edges=None, neighbor_mask=None):
    """Node digests of the prefix cache (se3_prefix_keys_fwd, DESIGN.md 10.4) of rows concatenated per cloud: feats [M, W]
    float32, each row's conv_in input with its degrees flattened and concatenated; coors [M, 3] float32; seqlens and n_prev (default
    zeros) per cloud; edges None or one [m_c, n_cur_c] int64 token or [m_c, n_cur_c, edge_dim] float32 tensor per cloud;
    neighbor_mask None or one bool [m_c, n_cur_c] per cloud.  Node i of a cloud covers columns j < i of its pair rows only.
    Returns int64 [M, 2]: the bits of each node's two uint64 lanes.  The descriptors go up in one copy; nothing is read back."""
    if feats.dtype != torch.float32 or feats.dim() != 2 or coors.dtype != torch.float32 or tuple(coors.shape) != (feats.shape[0], 3):
        raise ValueError('prefix_keys: feats must be float32 [M, W] and coors float32 [M, 3]')
    masks = list(neighbor_mask) if neighbor_mask is not None else None
    pairs = list(edges) if edges is not None else None
    _require_cuda(feats, coors, *(masks or ()), *(pairs or ()))
    seqlens = [int(m) for m in seqlens]
    n_prev = [0] * len(seqlens) if n_prev is None else [int(p) for p in n_prev]
    M, B = feats.shape[0], len(seqlens)
    if B == 0 or len(n_prev) != B or min(seqlens) < 1 or min(n_prev) < 0 or sum(seqlens) != M:
        raise ValueError(f'prefix_keys: need one seqlen >= 1 and n_prev >= 0 per cloud, summing to the {M} rows')
    if M >= 2 ** 31:
        raise ValueError(f'prefix_keys: {M} rows exceed the 1-D grid')
    n_cur = [p + m for p, m in zip(n_prev, seqlens)]
    off, at = [], 0                               # the pair rows of every cloud, [m_c, n_cur_c] entries each, end to end
    for m, n in zip(seqlens, n_cur):
        off.append(at)
        at += m * n
    nbr = None
    if masks is not None:
        if len(masks) != B or any(t is None or tuple(t.shape) != (m, n) for t, m, n in zip(masks, seqlens, n_cur)):
            raise ValueError(f'prefix_keys: neighbor_mask must be a list of {B} per-cloud [m, n_cur] masks')
        nbr = torch.cat([_u8(t).reshape(-1) for t in masks])
    tokens = values = None
    edge_dim = 0
    if pairs is not None:
        if len(pairs) != B:
            raise ValueError(f'prefix_keys: edges must be a list of {B} per-cloud tensors')
        floating = pairs[0].is_floating_point()
        for c, t in enumerate(pairs):
            want = torch.float32 if floating else torch.int64
            if t.dtype != want or tuple(t.shape[:2]) != (seqlens[c], n_cur[c]) or t.dim() != (3 if floating else 2):
                raise ValueError(f'prefix_keys: edges[{c}] must be {"float32 [m, n_cur, edge_dim]" if floating else "int64 [m, n_cur]"} '
                                 f'with [m, n_cur] = {[seqlens[c], n_cur[c]]}, got {t.dtype} {tuple(t.shape)}')
        flat = torch.cat([t.contiguous().reshape(-1) for t in pairs])
        if floating:
            values, edge_dim = flat, int(pairs[0].shape[2])
        else:
            tokens = flat
    cu = [0]
    for m in seqlens:
        cu.append(cu[-1] + m)
    dev = feats.device
    desc = torch.tensor(cu + n_prev + off, dtype=torch.int64).to(dev)
    feats, coors = feats.contiguous(), coors.contiguous()
    out = torch.empty((M, 2), dtype=torch.int64, device=dev)
    nbytes = 4 * feats.numel() + 12 * M + sum(t.numel() * t.element_size() for t in (tokens, values, nbr) if t is not None)
    with torch.cuda.device(dev), _timed('prefix_keys', nbytes=nbytes):
        _check(lib().se3_prefix_keys_fwd(_p(feats), M, feats.shape[1], _p(coors), _p(tokens), _p(values), edge_dim, _p(nbr),
                                         _p(desc[:B + 1]), _p(desc[B + 1:2 * B + 1]),
                                         _p(desc[2 * B + 1:]) if (pairs is not None or nbr is not None) else None, B, _p(out),
                                         _stream()))
    return out


def gather_pairs(pair_feat, idx):
    """pair_feat [b,n,n,e] -> [b,n,k,e] (reference utils.py:56-70 at S:1293-1294)."""
    _require_cuda(pair_feat, idx)
    pair_feat = _f32(pair_feat)
    b, n, _, e = pair_feat.shape
    k = idx.shape[-1]
    out = torch.empty((b, n, k, e), dtype=torch.float32, device=pair_feat.device)
    with torch.cuda.device(pair_feat.device):
        _check(lib().se3_gather_pairs_fwd(_p(pair_feat), _p(idx.contiguous()), b, n, k, e, _p(out), _stream()))
    return out


# ---------------------------------------------------------------------------------------------------------
# K2
# ---------------------------------------------------------------------------------------------------------
_QJ = None


def qj_table(J, d_in, d_out):
    """Q_J tables (reference basis.py:123-138), shipped as data generated by the reference routine so that the sign
    convention matches trained reference weights (SURVEY.md finding 6)."""
    global _QJ
    if _QJ is None:
        _QJ = dict(np.load(os.path.join(_PKG, 'data', 'qj_tables.npz')))
    return _QJ[f'{J}_{d_in}_{d_out}']


MAX_DEGREE = 5


class BasisPlan:
    """CSR view of all Q_J tables for one max_degree + the per-pair output layout."""
    _cache = {}

    def __init__(self, max_degree, device):
        if max_degree > MAX_DEGREE:
            raise ValueError(f'max_degree {max_degree} > {MAX_DEGREE} (Q_J tables shipped up to degree {MAX_DEGREE})')
        self.max_degree = max_degree
        self.pairs = [(di, do) for di in range(max_degree + 1) for do in range(max_degree + 1)]
        row_ptr, col, val = [0], [], []
        pair_row0, pair_base = [0], []
        base = 0
        for di, do in self.pairs:
            P, Q, F = 2 * do + 1, 2 * di + 1, 2 * min(di, do) + 1
            tabs = [qj_table(abs(di - do) + f, di, do) for f in range(F)]
            for pq in range(P * Q):
                for f in range(F):
                    J = abs(di - do) + f
                    row = tabs[f][pq]
                    thr = 1e-6 * np.abs(tabs[f]).max()
                    for m in np.nonzero(np.abs(row) > thr)[0]:
                        col.append(J * J + int(m))
                        val.append(float(row[m]))
                    row_ptr.append(len(col))
            pair_base.append(base)
            base += P * Q * F
            pair_row0.append(pair_row0[-1] + P * Q * F)
        self.rows_per_edge = base
        self.pair_base = pair_base
        self.pair_rows = [pair_row0[i + 1] - pair_row0[i] for i in range(len(self.pairs))]
        mk = lambda a, dt: torch.tensor(a, dtype=dt, device=device)
        self.row_ptr, self.col, self.val = mk(row_ptr, torch.int32), mk(col, torch.int32), mk(val, torch.float32)
        self.pair_row0, self.pair_base_t = mk(pair_row0, torch.int32), mk(pair_base, torch.int32)

    @classmethod
    def get(cls, max_degree, device):
        key = (max_degree, str(device))
        if key not in cls._cache:
            cls._cache[key] = cls(max_degree, device)
        return cls._cache[key]


def basis_flat(rel_pos, max_degree):
    """rel_pos [..., 3] -> (flat fp32 buffer, plan); pair p lives at flat[base_p*E : (base_p+rows_p)*E] as [E, rows_p]."""
    _require_cuda(rel_pos)
    rel_pos = _f32(rel_pos)
    E = rel_pos.numel() // 3
    plan = BasisPlan.get(max_degree, rel_pos.device)
    out = torch.empty(plan.rows_per_edge * E, dtype=torch.float32, device=rel_pos.device)
    with torch.cuda.device(rel_pos.device), _timed('basis', nbytes=E * (12 + 4 * plan.rows_per_edge)):
        _check(lib().se3_basis_fwd(_p(rel_pos), E, max_degree, _p(plan.row_ptr), _p(plan.col), _p(plan.val),
                                   _p(plan.pair_row0), _p(plan.pair_base_t), len(plan.pairs), _p(out), _stream()))
    return out, plan


def get_basis(r_ij, max_degree, differentiable=False):
    """Drop-in for the reference get_basis (basis.py:153-205): {'di,do': [..., 1, 2do+1, 1, 2di+1, f]} (forward only)."""
    flat, plan = basis_flat(r_ij, max_degree)
    E = r_ij.numel() // 3
    lead = tuple(r_ij.shape[:-1])
    out = {}
    for (di, do), base, rows in zip(plan.pairs, plan.pair_base, plan.pair_rows):
        out[f'{di},{do}'] = flat[base * E:(base + rows) * E].view(*lead, 1, 2 * do + 1, 1, 2 * di + 1, 2 * min(di, do) + 1)
    return out


def basis_pairs(flat, plan, E):
    """{(di,do): [E, P, Q, F] view} on the flat buffer."""
    out = {}
    for (di, do), base, rows in zip(plan.pairs, plan.pair_base, plan.pair_rows):
        out[(di, do)] = flat[base * E:(base + rows) * E]
    return out


# ---------------------------------------------------------------------------------------------------------
# K3 / K4
# ---------------------------------------------------------------------------------------------------------
RADIAL_MID = 128
TILE_E, TILE_O, TILE_IF = 128, 32, 4


def trunk_param_stride(in_dim):
    return in_dim * RADIAL_MID + 3 * RADIAL_MID + RADIAL_MID * RADIAL_MID + 3 * RADIAL_MID


def radial_trunk(feat, params, num_pairs):
    """feat [E, in_dim], params [num_pairs, trunk_param_stride] -> g [pairs, E, 128] fp32."""
    _require_cuda(feat, params)
    feat = _f32(feat)
    E, in_dim = feat.shape
    g = torch.empty((num_pairs, E, RADIAL_MID), dtype=torch.float32, device=feat.device)
    with torch.cuda.device(feat.device), _timed('radial_trunk', flops=2 * E * num_pairs * RADIAL_MID * (in_dim + RADIAL_MID),
                                                 nbytes=4 * (feat.numel() + params.numel() + g.numel())):
        _check(lib().se3_radial_trunk_fwd(_p(feat), E, in_dim, num_pairs, _p(params), _p(g), _stream()))
    return g


def t_numel(num_tiles, Ci, F, P):
    nifb = (Ci * F + TILE_IF - 1) // TILE_IF
    ph = (P + 3) // 4
    return num_tiles * nifb * TILE_IF * ph * TILE_E * 4


def _tile_range(E, tile_begin, tile_count):
    """(tile_count, edges) of a launch over tiles tile_begin .. tile_begin + tile_count of E edges (None: to the last tile)."""
    if tile_count is None:
        tile_count = (E + TILE_E - 1) // TILE_E - tile_begin
    return tile_count, min(E - tile_begin * TILE_E, tile_count * TILE_E)


def _tbuild_launch(x, idx, blocks, P, F, tile_begin, tile_count, out, flops, nbytes):
    """se3_tbuild_fwd into `out` (reallocated if missing or too small): x [b,n,Ci,Q] fp32, blocks [E,P,Q,F] flat."""
    b, n, Ci, Q = x.shape
    numel = t_numel(tile_count, Ci, F, P)
    if out is None or out.numel() < numel:
        out = torch.empty(numel, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device), _timed('tbuild', flops=flops, nbytes=nbytes):
        _check(lib().se3_tbuild_fwd(_p(x), _p(idx.contiguous()), _p(blocks), b, n, idx.shape[-1], Ci, P, Q, F, tile_begin, tile_count,
                                    _p(out), _stream()))
    return out


def tbuild(x, idx, basis_pair, d_in, d_out, tile_begin=0, tile_count=None, out=None):
    """x [b,n,Ci,2di+1], idx [b,n,k], basis_pair flat [E*P*Q*F] -> T (tile layout, see include/se3b200.h)."""
    return tbuild_blocks(x, idx, basis_pair, 2 * d_out + 1, 2 * min(d_in, d_out) + 1, tile_begin, tile_count, out)


_IDENTITY_BASIS = {}


def gather_tiles(x, idx, tile_begin=0, tile_count=None, out=None):
    """Neighbour features in the T tile layout: X[e,i,q] = x[b, idx[e], i, q] (se3_tbuild_fwd with an identity basis,
    P := Q, F := 1); the right-hand operand of the input-side contraction."""
    _require_cuda(x, idx)
    x = _f32(x)
    b, n, Ci, Q = x.shape
    E = b * n * idx.shape[-1]
    key = (E, Q, x.device)
    if key not in _IDENTITY_BASIS:
        _IDENTITY_BASIS.clear()
        _IDENTITY_BASIS[key] = torch.eye(Q, dtype=torch.float32, device=x.device).repeat(E, 1, 1).reshape(-1).contiguous()
    tile_count, Ec = _tile_range(E, tile_begin, tile_count)
    return _tbuild_launch(x, idx, _IDENTITY_BASIS[key], Q, 1, tile_begin, tile_count, out, flops=2 * Ec * Ci * Q * Q,
                          nbytes=4 * Ec * (2 * Ci * Q) + 8 * Ec)


def tbuild_blocks(x, idx, blocks, P, F, tile_begin=0, tile_count=None, out=None):
    """se3_tbuild_fwd with caller-supplied per-edge blocks [E,P,Q,F] (flat): T[e,i,f,p] = sum_q blocks[e,p,q,f] x[b, idx[e], i, q]."""
    _require_cuda(x, idx, blocks)
    x = _f32(x)
    b, n, Ci, Q = x.shape
    E = b * n * idx.shape[-1]
    assert blocks.numel() == E * P * Q * F
    tile_count, Ec = _tile_range(E, tile_begin, tile_count)
    # bytes WITHOUT the layout padding of T
    return _tbuild_launch(x, idx, blocks, P, F, tile_begin, tile_count, out, flops=2 * Ec * Ci * F * P * Q,
                          nbytes=4 * Ec * (Ci * F * P + P * Q * F + Ci * Q) + 8 * Ec)


def fold_basis(S, basis_pair, E, Co, P, Q, F, out, accumulate, component_major=False, name='fold_basis'):
    """out [E,Co,P] (+)= sum_{f,q} basis_pair[e,p,q,f] S[f,e,o,q]; S [F,E,Co,Q] (or [F,E,Q,Co] if component_major),
    basis_pair the [E,P,Q,F] rows of these edges."""
    _require_cuda(S, basis_pair, out)
    assert S.is_contiguous() and basis_pair.is_contiguous() and out.is_contiguous()
    nbytes = 4 * (S.numel() + basis_pair.numel() + out.numel() * (2 if accumulate else 1))
    with torch.cuda.device(out.device), _timed(name, flops=2 * E * Co * P * Q * F, nbytes=nbytes):
        fn = lib().se3_fold_basis_cm_fwd if component_major else lib().se3_fold_basis_fwd
        _check(fn(_p(S), _p(basis_pair), E, Co, P, Q, F, int(accumulate), _p(out), _stream()))


def rotate_back(parts, D, E, Co, lo, out):
    """out [E,Co,2lo+1] = D_lo(e) out'(e): parts[0] [E,Co] (m = 0), parts[m] [E,Co,2] (components +m, -m) or None."""
    _require_cuda(D, out, *parts)
    ptrs = [(_p(t) if t is not None else None) for t in (list(parts) + [None] * 4)[:4]]
    P = 2 * lo + 1
    nbytes = 4 * (2 * E * Co * P + E * P * P)
    with torch.cuda.device(out.device), _timed('rotate_back', flops=2 * E * Co * P * P, nbytes=nbytes):
        _check(lib().se3_rotate_back_fwd(*ptrs, _p(D), E, Co, lo, _p(out), _stream()))


def pairwise_simt(g, W3, b3, T, E, Co, Ci, F, P, out, accumulate):
    _require_cuda(g, W3, b3, T, out)
    with torch.cuda.device(out.device), _timed('pairwise_simt', flops=2 * E * Co * Ci * F * (RADIAL_MID + P), fma=2 * E * Co * Ci * F * (RADIAL_MID + P)):
        _check(lib().se3_pairwise_simt_fwd(_p(g), _p(W3), _p(b3), _p(T), E, Co, Ci, F, P, int(accumulate), _p(out), _stream()))


def w3_image_bytes(Co, Ci, F):
    return lib().se3_w3_image_bytes(Co, Ci, F)


def pack_w3(W3, b3, Co, Ci, F):
    _require_cuda(W3, b3)
    nbytes = w3_image_bytes(Co, Ci, F)
    if nbytes < 0:
        raise RuntimeError(f'pack_w3: unsupported shape Co={Co} Ci={Ci} F={F}')
    img = torch.empty(nbytes, dtype=torch.uint8, device=W3.device)
    with torch.cuda.device(W3.device):
        _check(lib().se3_pack_w3(_p(_f32(W3)), _p(_f32(b3)), Co, Ci, F, _p(img), _stream()))
    return img


def pairwise_tc(g, w_img, T, E, Co, Ci, F, P, out, accumulate, dump=None):
    _require_cuda(g, w_img, T, out)
    # algorithmic work: the radial GEMM (2*128 per R element) + the contraction with T (2*P per R element)
    flops = 2 * E * Co * Ci * F * (RADIAL_MID + P)
    nbytes = w_img.numel() + 4 * E * Ci * F * P + 4 * E * Co * P * (2 if accumulate else 1)
    with torch.cuda.device(out.device), _timed('pairwise_tc', flops=flops, nbytes=nbytes, tag=f'P{P}F{F}Ci{Ci}Co{Co}',
                                               mma=2 * E * Co * Ci * F * 3 * RADIAL_MID, fma=2 * E * Co * Ci * F * P):
        if dump is None:
            _check(lib().se3_pairwise_tc_fwd(_p(g), _p(w_img), _p(T), E, Co, Ci, F, P, int(accumulate), _p(out), _stream()))
        else:
            _check(lib().se3_pairwise_tc_debug(_p(g), _p(w_img), _p(T), E, Co, Ci, F, P, int(accumulate), _p(out), _p(dump),
                                               _stream()))


def pack_lowrank(Fp, Co, Ci, F, Kp):
    """Fp [Co*Ci*F, Kp] fp32 (W3 V | b3 | 0) -> tensor-core operand image for pairwise_lr."""
    _require_cuda(Fp)
    nbytes = lib().se3_lowrank_image_bytes(Co, Ci, F, Kp)
    if nbytes < 0:
        raise RuntimeError(f'pack_lowrank: unsupported shape Co={Co} Ci={Ci} F={F}')
    img = torch.empty(nbytes, dtype=torch.uint8, device=Fp.device)
    with torch.cuda.device(Fp.device):
        _check(lib().se3_pack_lowrank(_p(_f32(Fp)), Co, Ci, F, Kp, _p(img), _stream()))
    return img


def pairwise_lr(U, w_img, T, E, Co, Ci, F, P, Kp, out, accumulate, alg_P=None, alg_units=None):
    """Low-rank radial path: U [E,64] fp32 (G V | 1 | 0), w_img from pack_lowrank."""
    _require_cuda(U, w_img, T, out)
    # algorithmic work of the reference formulation (SURVEY.md 8d): 2*128 (radial GEMM) + 2P (contraction) per R element;
    # executed work: the GEMM has K = Kp instead of 128
    # (alg_P: the launch is one frequency of an input-side contraction whose reference formulation has P = alg_P)
    # (alg_units: reference-formulation FLOPs per (edge, o, i) that this launch stands for, when it is not F*(2*128 + 2P))
    flops = 2 * E * Co * Ci * F * (RADIAL_MID + (alg_P if alg_P is not None else P))
    if alg_units is not None:
        flops = E * Co * Ci * alg_units
    # issued: 3 fp16 MMA passes of K = Kp per R element on the tensor cores, P fp32 FMAs per R element on the SIMT pipe
    nbytes = w_img.numel() + 4 * E * Ci * F * P + 4 * E * Co * P * (2 if accumulate else 1)
    tag = f'P{P}F{F}Ci{Ci}Co{Co}K{Kp}' + (f'(in-side of P{alg_P})' if alg_P is not None else '')
    with torch.cuda.device(out.device), _timed('pairwise_lr', flops=flops, nbytes=nbytes, tag=tag,
                                               mma=2 * E * Co * Ci * F * 3 * Kp, fma=2 * E * Co * Ci * F * P):
        _check(lib().se3_pairwise_lr_fwd(_p(U), _p(w_img), _p(T), E, Co, Ci, F, P, Kp, int(accumulate), _p(out), _stream()))


# ---------------------------------------------------------------------------------------------------------
# production path: low-rank radial basis + edge-aligned frames as one GEMM per (degree_out, |m|)  (csrc/zgemm.cu, aligned.cu)
# ---------------------------------------------------------------------------------------------------------
class ZSeg(ctypes.Structure):
    _fields_ = [('U', c_void_p), ('X', c_void_p), ('Ci', c_int), ('ncomp', c_int), ('cplus', c_int), ('cminus', c_int)]


def radial_trunk_u(feat, params, V, gmean, ones_col, stats, want_g=False):
    """Trunk + radial coordinates: feat [E,in_dim], params [pairs, stride], V [pairs,128,64] fp32, gmean [pairs,128] fp32 (centre of
    the pair's radial curve), ones_col [pairs] int32, stats [pairs,2] fp32 (accumulates (max residual, max |g|)) ->
    U [pairs,E,64] = ((g - gmean) V | 1 | 0) (, g [pairs,E,128])."""
    _require_cuda(feat, params, V, gmean, ones_col, stats)
    assert gmean.shape == (params.shape[0], RADIAL_MID) and gmean.is_contiguous() and gmean.dtype == torch.float32
    feat = _f32(feat)
    E, in_dim = feat.shape
    num_pairs = params.shape[0]
    assert V.shape == (num_pairs, RADIAL_MID, 64) and V.is_contiguous() and ones_col.dtype == torch.int32 and stats.is_contiguous()
    U = torch.empty((num_pairs, E, 64), dtype=torch.float32, device=feat.device)
    g = torch.empty((num_pairs, E, RADIAL_MID), dtype=torch.float32, device=feat.device) if want_g else None
    flops = 2 * E * num_pairs * RADIAL_MID * (in_dim + RADIAL_MID + 2 * 64)
    with torch.cuda.device(feat.device), _timed('radial_trunk', flops=flops, nbytes=4 * (feat.numel() + params.numel() + V.numel() + U.numel())):
        _check(lib().se3_radial_trunk_u_fwd(_p(feat), E, in_dim, num_pairs, _p(params), _p(V), _p(gmean), _p(ones_col), _p(g), _p(U), _p(stats), _stream()))
    return U, g


def radial_table(dist, table, Dmax, ones_col, stats):
    """Radial coordinates by table lookup: dist [E] fp32, table [pairs, G, KT] fp32 (U(d) on the uniform grid of [0, Dmax]),
    ones_col [pairs] int32, stats [pairs, 2] (out-of-range flag) -> U [pairs, E, 64]."""
    _require_cuda(dist, table, ones_col, stats)
    dist = _f32(dist).reshape(-1)
    E = dist.numel()
    num_pairs, G, KT = table.shape
    assert table.is_contiguous() and table.dtype == torch.float32 and ones_col.dtype == torch.int32
    U = torch.empty((num_pairs, E, 64), dtype=torch.float32, device=dist.device)
    with torch.cuda.device(dist.device), _timed('radial_table', flops=8 * E * num_pairs * KT, nbytes=4 * (E + U.numel() + 4 * E * num_pairs * KT)):
        _check(lib().se3_radial_table_fwd(_p(dist), E, _p(table), G, KT, float(Dmax), _p(ones_col), num_pairs, _p(U), _p(stats), _stream()))
    return U


_FRAME_TABLES = {}


def _frame_tables(lmax, device):
    key = (lmax, str(device))
    if key not in _FRAME_TABLES:
        from . import aligned
        xs_t, pin_t, keep = [None], [None], []
        ns = [0]
        for l in range(1, lmax + 1):
            xs, pin = aligned._samples(l, device)
            xs, pin = xs.contiguous(), pin.contiguous()
            keep += [xs, pin]
            xs_t.append(xs.data_ptr()); pin_t.append(pin.data_ptr()); ns.append(xs.shape[0])
        mk = lambda vals: (c_void_p * (lmax + 1))(*[c_void_p(v) if v else None for v in vals])
        _FRAME_TABLES[key] = (mk(xs_t), mk(pin_t), (c_int * (lmax + 1))(*ns), keep)
    return _FRAME_TABLES[key]


def frames(rel_pos, lmax):
    """Wigner matrices of the edge frames: rel_pos [...,3] -> [None, D_1 [E,3,3], ..., D_lmax] fp32 (float64 arithmetic inside)."""
    _require_cuda(rel_pos)
    rel_pos = _f32(rel_pos).reshape(-1, 3)
    E = rel_pos.shape[0]
    D = [None] + [torch.empty((E, 2 * l + 1, 2 * l + 1), dtype=torch.float32, device=rel_pos.device) for l in range(1, lmax + 1)]
    if lmax >= 1:
        xs, pin, ns, _ = _frame_tables(lmax, rel_pos.device)
        dptr = (c_void_p * (lmax + 1))(*[c_void_p(t.data_ptr()) if t is not None else None for t in D])
        with torch.cuda.device(rel_pos.device), _timed('frames', nbytes=E * (12 + 4 * sum((2 * l + 1) ** 2 for l in range(1, lmax + 1)))):
            _check(lib().se3_frames_fwd(_p(rel_pos), E, lmax, xs, pin, ns, dptr, _stream()))
    return D


def rotgather(x, idx, D, tile_begin=0, tile_count=None, out=None):
    """x [b,n,Ci,Q], idx [b,n,k], D [E,Q,Q] (None for Q = 1) -> X [tile_count, Ci, Q, 128]: rotated neighbour features."""
    _require_cuda(x, idx, D)
    x = _f32(x)
    b, n, Ci, Q = x.shape
    k = idx.shape[-1]
    tile_count, Ec = _tile_range(b * n * k, tile_begin, tile_count)
    numel = tile_count * Ci * Q * TILE_E
    if out is None or out.numel() < numel:
        out = torch.empty(numel, dtype=torch.float32, device=x.device)
    nbytes = 4 * Ec * (2 * Ci * Q + (Q * Q if Q > 1 else 0)) + 8 * Ec
    with torch.cuda.device(x.device), _timed('rotgather', flops=2 * Ec * Ci * Q * Q, nbytes=nbytes):
        _check(lib().se3_rotgather_fwd(_p(x), _p(idx.contiguous()), _p(D), b, n, k, Ci, Q, tile_begin, tile_count, _p(out), _stream()))
    return out


def rotate_pool(Op, D, mask, self_add, nodes, K, Co, lo, out):
    """Pooled ConvSE3 epilogue fused with the rotate-back: Op [nodes*K, 2lo+1, Co], D [nodes*K, P, P] or None (lo = 0),
    mask [nodes*K] bool or None, self_add [nodes, Co, P] or None -> out [nodes, Co, P]."""
    _require_cuda(Op, D, mask, self_add, out)
    P = 2 * lo + 1
    assert Op.is_contiguous() and out.is_contiguous() and (self_add is None or self_add.is_contiguous())
    nbytes = 4 * (Op.numel() + out.numel() * (2 if self_add is not None else 1) + (nodes * K * P * P if lo else 0)) + nodes * K
    with torch.cuda.device(out.device), _timed('rotate_pool', flops=2 * nodes * K * Co * P * P, nbytes=nbytes):
        _check(lib().se3_rotate_pool_fwd(_p(Op), _p(D), _p(_u8(mask)), _p(self_add), nodes, K, Co, lo, _p(out), _stream()))


def node_absmax(feats):
    """The largest |component| of every node's features over all degrees: feats {d: [b, n, C, 2d+1]} -> [b * n] fp32."""
    first = True
    for t in feats.values():
        t = _f32(t)
        if first:
            rows = t.shape[0] * t.shape[1]
            nodemax = torch.empty(rows, dtype=torch.float32, device=t.device)
        with torch.cuda.device(t.device):
            _check(lib().se3_rowabsmax_fwd(_p(t), rows, t.shape[2] * t.shape[3], int(not first), _p(nodemax), _stream()))
        first = False
    return nodemax


def edge_scale(feats, idx, max_degree, nodemax=None):
    """Power-of-two scale per edge from the largest |component| of the neighbour's features (all degrees): [E] fp32.  With
    nodemax (node_absmax of every node idx addresses, [b * n]) feats is not read."""
    b, n, k = idx.shape
    if nodemax is None:
        nodemax = node_absmax(feats)
    with torch.cuda.device(idx.device):
        sx = torch.empty(b * n * k, dtype=torch.float32, device=idx.device)
        _check(lib().se3_edge_scale_fwd(_p(nodemax), _p(idx.contiguous()), b, n, k, max_degree, _p(sx), _stream()))
    return sx


def linear_supported(D, Eo, device):
    """Shapes the tensor-core LinearSE3 kernel takes."""
    return D % 64 == 0 and Eo % 128 == 0 and torch.cuda.get_device_capability(device) == (9, 0)


def linear_image(W):
    """W [D, Eo] fp32 (LinearSE3.weights[degree]) -> tensor-core operand image of W^T for linear_tc."""
    _require_cuda(W)
    D, Eo = W.shape
    Fp = _f32(W.detach().t()).contiguous().reshape(Eo * (D // 16), 16)
    nbytes = lib().se3_zgemm_image_bytes(Eo, 4, D // 64)
    if nbytes < 0:
        raise RuntimeError(f'linear_image: unsupported shape D={D} Eo={Eo}')
    img = torch.empty(nbytes, dtype=torch.uint8, device=W.device)
    with torch.cuda.device(W.device):
        _check(lib().se3_zgemm_pack(_p(Fp), 16, 0, Eo, D // 16, 4, D // 64, 0, _p(img), _stream()))
    return img


def linear_tc(x, img, Eo, res=None, flush_stages=0):
    """LinearSE3 on the tensor cores: x [b,n,D,M] (reference layout, read in place) -> [b,n,Eo,M] (+ res); the fp32 partial
    sums are drained every flush_stages stages (0: the library's default)."""
    _require_cuda(x, img, res)
    x = _f32(x)
    b, n, D, M = x.shape
    nodes = b * n
    out = torch.empty((b, n, Eo, M), dtype=torch.float32, device=x.device)
    if res is not None:
        res = _f32(res)
        assert res.shape == out.shape
    with torch.cuda.device(x.device):
        rowmax = torch.empty(nodes, dtype=torch.float32, device=x.device)
        sx = torch.empty(nodes, dtype=torch.float32, device=x.device)
        _check(lib().se3_rowabsmax_fwd(_p(x), nodes, D * M, 0, _p(rowmax), _stream()))
        _check(lib().se3_pow2_scale_fwd(_p(rowmax), nodes, 14, _p(sx), _stream()))
        nbytes = img.numel() + 4 * (2 * x.numel() + out.numel() * (2 if res is not None else 1))
        with _timed('linear', flops=2 * nodes * M * D * Eo, nbytes=nbytes, mma=2 * nodes * M * D * Eo * 3, tag=f'linear D{D}E{Eo}M{M}'):
            _check(lib().se3_linear_tc_fwd(_p(x), _p(img), _p(res), _p(sx), nodes, D, Eo, M, _p(out), flush_stages, _stream()))
    return out


def zgemm_tile_n(Co, mode):
    return lib().se3_zgemm_tile_n(Co, mode)


def zgemm_image(parts, Co, mode):
    """parts: [(Fp [Co*Ci*F, Kp] fp32, Ci)] in K order (one entry per input degree; Kp / 16 sub-segments each; F = 1 for mode 1,
    rows (o, i, (a, b)) for modes 2 and 3) -> (uint8 image, total_stages)."""
    F = 1 if mode == 1 else 2
    per_seg = (lambda Ci: 3 * (Ci // 4)) if mode == 3 else (lambda Ci: Ci * F // 4)
    stages = [(Fp.shape[1] // 16) * per_seg(Ci) for Fp, Ci in parts]
    S = sum(stages)
    nbytes = lib().se3_zgemm_image_bytes(Co, mode, S)
    if nbytes < 0:
        raise RuntimeError(f'zgemm_image: unsupported shape Co={Co} mode={mode}')
    dev = parts[0][0].device
    img = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    s0 = 0
    with torch.cuda.device(dev):
        for Fp, Ci in parts:
            _require_cuda(Fp)
            Fp = _f32(Fp)
            Kp = Fp.shape[1]
            assert Fp.shape[0] == Co * Ci * F and Kp % 16 == 0 and (Ci * F) % 4 == 0
            for kc in range(Kp // 16):
                _check(lib().se3_zgemm_pack(_p(Fp), Kp, 16 * kc, Co, Ci * F, mode, S, s0, _p(img), _stream()))
                s0 += per_seg(Ci)
    return img, S


SPLIT_LAUNCHES = 0    # zgemm launches of this process that ran split-K (k_split > 1)
_SMS = {}


def sm_count(device):
    """Streaming multiprocessors of `device`."""
    key = torch.device(device).index if torch.device(device).index is not None else torch.cuda.current_device()
    if key not in _SMS:
        _SMS[key] = torch.cuda.get_device_properties(key).multi_processor_count
    return _SMS[key]


def zgemm_k_split(tiles, units, sms):
    """CTAs per output tile of a zgemm launch with `tiles` output tiles and `units` split units on a card of `sms` SMs: 1 when the
    unsplit grid already has a CTA per SM, else as many as fit one wave, at most one unit each."""
    if tiles >= sms:
        return 1
    return max(1, min(units, sms // tiles))


def zgemm(segs, w_img, sx, E, Co, mode, out, out_edge_stride, comp_off, flush_stages=0, alg_flops=0, tag='', k_split=None):
    """segs: [(U [E,64] view (row stride 64; column offset folded into the pointer), X buffer, Ci, ncomp, cplus, cminus)].
    k_split: CTAs per output tile (split-K over whole drain / Gauss blocks, bit-identical to 1); None chooses it from the grid,
    the launch's split units and the SM count (zgemm_k_split).  A forced value above the launch's units is refused."""
    global SPLIT_LAUNCHES
    _require_cuda(w_img, sx, out)
    arr = (ZSeg * len(segs))()
    Ktot = 0
    for i, (U, X, Ci, ncomp, cplus, cminus) in enumerate(segs):
        _require_cuda(U, X)
        assert U.dtype == torch.float32 and U.stride(-1) == 1 and (U.dim() == 1 or U.stride(0) == 64)
        arr[i] = ZSeg(U.data_ptr(), X.data_ptr(), Ci, ncomp, cplus, cminus)
        Ktot += Ci * (1, 2, 3)[mode - 1] * 16
    N = zgemm_tile_n(Co, mode)
    # issued tensor-core FLOPs: 3 fp16 passes of 2 M N K; mode 2 feeds two accumulators from every B tile, mode 3 has three
    # weight sets with one accumulator each
    mma = 2 * E * Co * Ktot * 3 * (2 if mode == 2 else 1)
    planes = 1 if mode == 1 else 2
    nbytes = w_img.numel() + 4 * E * Co * planes + sum(4 * E * s[2] * (planes + 16) for s in segs)
    units = lib().se3_zgemm_split_units(arr, len(segs), Co, mode, flush_stages)
    if units < 1:
        raise ValueError(f'zgemm: unsupported launch (Co={Co}, mode={mode}, {len(segs)} segments)')
    if k_split is None:
        k_split = zgemm_k_split(((E + TILE_E - 1) // TILE_E) * (Co // (64 if mode == 2 else 128)), units, sm_count(out.device))
    elif not 1 <= k_split <= units:
        raise ValueError(f'zgemm: k_split = {k_split} outside [1, {units}], the split units (drain / Gauss blocks) of this launch')
    ws, ws_bytes = None, 0
    if k_split > 1:
        ws_bytes = lib().se3_zgemm_workspace_bytes(arr, len(segs), E, Co, mode, flush_stages)
        ws = torch.empty(ws_bytes // 4, dtype=torch.float32, device=out.device)
        SPLIT_LAUNCHES += 1
    tag = (tag or f'mode{mode}N{N}K{Ktot}') + (f'split{k_split}' if k_split > 1 else '')
    with torch.cuda.device(out.device), _timed('zgemm', flops=alg_flops, nbytes=nbytes, tag=tag, mma=mma):
        _check(lib().se3_zgemm_split_fwd(arr, len(segs), _p(w_img), _p(sx), E, Co, mode, _p(out), out_edge_stride, comp_off[0],
                                         comp_off[1] if len(comp_off) > 1 else 0, flush_stages, k_split, _p(ws), ws_bytes, _stream()))


# max-abs residual of the radial basis relative to max|G|.  The fp32 trunk itself carries ~6e-7..1e-6 of rounding noise
# against float64, so 1e-6 keeps the truncation below what fp32 can resolve; at the headline width (depth-2 slice of cfg2)
# the output differs from the fp32 SIMT path by 1.6e-5 with 1e-6 and by 1.5e-5 with 2e-7 or with the direct K = 128
# kernel.  With 1e-6, 96 % of the cfg2 pairs need rank <= 15 (K = 16) instead of 26 % with 2e-7.
LOWRANK_TOL = 1e-6


def lowrank_basis(G64, tol=LOWRANK_TOL, ranks=(15, 31, 47, 63)):
    """Affine low-rank model of the curve G64 [S, 128] (float64 samples of a radial trunk along its input curve):
    returns (r, V [128, r] float64 orthonormal, mean [128] float64) for the smallest listed rank with
    max|(G - mean) - ((G - mean) V) V^T| <= tol * max|G|, else None.  The mean costs nothing downstream: W3 mean joins the bias
    column of F' (the ones column of U), and centring lowers the rank the tolerance needs by one (measured on 120 random
    trunks: ranks 14/15/16/17 for 26/52/22/1 % without, 13/14/15/16 with), so that ~99 % instead of ~78 % of the pairs fit K = 16.
    QR + SVD of the triangular factor (no Gram matrix, so the small singular directions stay accurate)."""
    G64 = G64.detach()
    mean = G64.mean(dim=0)
    H = G64 - mean
    Rm = torch.linalg.qr(H, mode='r').R              # Q is never needed
    # SVD of the 128 x 128 triangular factor on the host: 128 KB to move, ~1 ms of LAPACK, instead of the hundreds of small
    # launches of the iterative device SVD per (degree_in, degree_out) pair at plan time
    Vh = torch.linalg.svd(Rm.cpu())[2].to(G64.device)
    gmax = float(G64.abs().max())
    for r in ranks:
        V = Vh[:r].t().contiguous()
        res = float((H - (H @ V) @ V.t()).abs().max())
        if res <= tol * gmax:
            return r, V, mean
    return None


def lowrank_enabled(E, sw=None):
    """A forward of E edges takes the low-rank radial path under the switches sw (default: switches.current())."""
    if sw is None:
        from .switches import current
        sw = current()
    return not sw.no_lowrank and E >= sw.lowrank_min_edges


def tc_supported(device, Co, P):
    """The wgmma kernel needs sm_90 and Co % 32 == 0, degree_out <= 3."""
    if Co % TILE_O != 0 or P > 7:
        return False
    return torch.cuda.get_device_capability(device) == (9, 0)


def pool(x, mask):
    """masked mean over axis 2 of x [b,n,k,...] with mask [b,n,k] (reference utils.py:72-80)."""
    _require_cuda(x, mask)
    x = _f32(x)
    b, n, k = x.shape[:3]
    C = x[0, 0, 0].numel()
    out = torch.empty((b, n) + tuple(x.shape[3:]), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device), _timed('pool', nbytes=4 * (x.numel() + out.numel()) + b * n * k):
        _check(lib().se3_pool_fwd(_p(x), _p(_u8(mask)), b * n, k, C, _p(out), _stream()))
    return out


# ---------------------------------------------------------------------------------------------------------
# K5
# ---------------------------------------------------------------------------------------------------------
ATTN_ALIGNED_MAX_DIM_HEAD = 128     # se3_attn_aligned_fwd keeps dim_head in at most 4 register slots per lane


def attn_aligned_supported(dim_head):
    """Heads the attention kernel with the fused rotate-back takes; wider heads rotate back separately and run se3_attn_fwd."""
    return dim_head <= ATTN_ALIGNED_MAX_DIM_HEAD


def attention(q, k, v, *, heads, dim_head, scale, nmask=None, k_idx=None, self_k=None, self_v=None, null_k=None, null_v=None,
              global_k=None, global_v=None, kv_heads=None, D=None, k_aligned=False):
    """One degree of AttentionSE3 / OneHeadedKVAttentionSE3 (reference S:476-517, 612-652).
    q [b,n,H*Dh,M]; k,v [b,n,K,Ckv,M] (k may be node level [b,n,Ckv,M] with k_idx [b,n,K]).
    With D [b*n*K, M, M] (edge frames): v (and k if k_aligned) are the edge-aligned, component-major [b,n,K,M,Ckv] outputs of
    zgemm and the rotation back to the global frame is fused into the kernel (se3_attn_aligned_fwd)."""
    _require_cuda(q, k, v, D)
    q, k, v = _f32(q), _f32(k), _f32(v)
    b, n, _, M = q.shape
    K = v.shape[2]
    kv_heads = heads if kv_heads is None else kv_heads
    G = 0 if global_k is None else global_k.shape[1]
    cont = lambda t: None if t is None else _f32(t)
    self_k, self_v, null_k, null_v, global_k, global_v = map(cont, (self_k, self_v, null_k, null_v, global_k, global_v))
    out = torch.empty_like(q)
    nm = _u8(nmask)
    ki = None if k_idx is None else k_idx.contiguous()
    J = K + G + (self_k is not None) + (null_k is not None)
    nbytes = 4 * (2 * q.numel() + 2 * b * n * J * heads * dim_head * M)
    if D is not None:
        assert M > 1 and D.is_contiguous() and D.numel() == b * n * K * M * M and v.shape[3] == M
        nbytes += 4 * D.numel()
        with torch.cuda.device(q.device), _timed('attention', flops=4 * b * n * J * heads * dim_head * M * (1 + M), nbytes=nbytes):
            _check(lib().se3_attn_aligned_fwd(_p(q), _p(k), _p(v), _p(D), int(bool(k_aligned)), _p(ki), _p(self_k), _p(self_v), _p(null_k),
                                              _p(null_v), _p(global_k), _p(global_v), G, _p(nm), b, n, K, heads, dim_head, M, kv_heads,
                                              float(scale), _p(out), _stream()))
        return out
    with torch.cuda.device(q.device), _timed('attention', flops=4 * b * n * J * heads * dim_head * M, nbytes=nbytes):
        _check(lib().se3_attn_fwd(_p(q), _p(k), _p(v), _p(ki), _p(self_k), _p(self_v), _p(null_k), _p(null_v), _p(global_k),
                                  _p(global_v), G, _p(nm), b, n, K, heads, dim_head, M, kv_heads, float(scale), _p(out), _stream()))
    return out


def norm_se3(x, scale, eps, use_gelu):
    """NormSE3 with a per-channel scale (reference S:130-152): x [b,n,C,M] -> same shape."""
    _require_cuda(x, scale)
    x = _f32(x)
    C, M = x.shape[-2], x.shape[-1]
    out = torch.empty_like(x)
    with torch.cuda.device(x.device), _timed('norm', nbytes=8 * x.numel()):
        _check(lib().se3_norm_fwd(_p(x), _p(_f32(scale).reshape(-1)), x.numel() // M, C, M, float(eps), int(use_gelu), _p(out), _stream()))
    return out
