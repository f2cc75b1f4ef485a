"""Shared helpers for the parity tests (no reference import; fixtures only)."""
import json
import os
import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')

MODEL_CASES = ['cfg1', 'deg4', 'af2', 'edges_sparse', 'ragged', 'tc_deg2', 'tc_deg4', 'allnbr', 'causal', 'tiekv',
               'linkeys', 'nullkv', 'noself', 'global', 'onehead', 'preconv_normout', 'tokens_pos', 'adjdeg', 'nbrmask',
               'contedges', 'rotary_both', 'rotary_pos_onehead', 'rotary_dist_linkeys', 'rotary_tiekv']

# BASELINE.json configs[2] at full size, configs[3] at batch 2 (the reference needs ~8 GB of host RAM per cloud there)
BIG_CASES = ['cfg3', 'cfg4_b2']


# widths the one-GEMM production kernel takes (every fiber a multiple of 128 channels, DESIGN.md 4.5)
Z_CASES = ['z128', 'z256_deg4']


def load_case(name):
    z = dict(np.load(os.path.join(GOLDEN, f'model_{name}.npz')))
    # the largest fixtures are split into model_<name>.part<i>.npz files (each stored file stays under 1 MB)
    for part in sorted(f for f in os.listdir(GOLDEN) if f.startswith(f'model_{name}.part')):
        z.update(np.load(os.path.join(GOLDEN, part)))
    cfg = json.loads(str(z.pop('config')))
    ctor = cfg['ctor']
    if isinstance(ctor.get('dim_in'), list):
        ctor['dim_in'] = tuple(ctor['dim_in'])
    return z, cfg


def state_keys(name):
    with open(os.path.join(GOLDEN, 'state_keys.json')) as f:
        return json.load(f)[name]


def det_params(name, seed=11):
    from detfill import det_tensor
    return {k: det_tensor(k, tuple(s), seed).astype(np.float32) for k, s in state_keys(name).items()
            if not k.endswith('inv_freq')}


def rel_err(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def case_inputs(z):
    inp = {k[3:]: v for k, v in z.items() if k.startswith('in/')}
    if 'feats' in inp:
        feats = inp['feats']
    else:
        feats = {'0': inp['feats/0'], '1': inp['feats/1']}
    extra = {k: inp[k] for k in ('adj_mat', 'edges', 'neighbor_mask', 'global_feats') if k in inp}
    return feats, inp['coors'], inp['mask'], extra


def case_outputs(z):
    if 'out' in z:
        return z['out']
    return {k[4:]: v for k, v in z.items() if k.startswith('out/')}


def assert_graph_equal(idx, mask, dist, ref_idx, ref_mask, ref_dist, atol=1e-5):
    """Neighbour lists agree as sets of valid (unmasked) neighbours with the same distances."""
    assert idx.shape == ref_idx.shape
    big = np.iinfo(np.int64).max
    a = np.where(mask, idx, big)
    b = np.where(ref_mask, ref_idx, big)
    oa = np.argsort(a, -1, kind='stable')
    ob = np.argsort(b, -1, kind='stable')
    assert np.array_equal(np.take_along_axis(a, oa, -1), np.take_along_axis(b, ob, -1))
    da = np.where(mask, dist, 0.0)
    db = np.where(ref_mask, ref_dist, 0.0)
    assert np.allclose(np.take_along_axis(da, oa, -1), np.take_along_axis(db, ob, -1), atol=atol)


# ---- layout decoders for the kernel-side images (DESIGN.md "data layout") ----
def decode_operand_image(img_u8):
    """uint8 [..., 65536] UMMA operand image -> (hi, lo) float32 [..., 128, 128] (rows, k)."""
    import torch
    img = img_u8.reshape(-1, 65536).cpu().numpy()
    as16 = img.view(np.uint16).reshape(img.shape[0], 2, 2, 128, 64)        # [tile][hi/lo][khalf][row][16B chunk * 8 + j]
    r = np.arange(128)[:, None]
    kk = np.arange(64)[None, :]
    phys = ((kk >> 3) ^ (r & 7)) * 8 + (kk & 7)                            # physical element index inside the 128-byte row
    out = np.empty((img.shape[0], 2, 128, 128), dtype=np.float32)
    for part in range(2):
        for kh in range(2):
            sub = np.take_along_axis(as16[:, part, kh], np.broadcast_to(phys, (img.shape[0], 128, 64)), axis=2)
            out[:, part, :, kh * 64:(kh + 1) * 64] = (sub.astype(np.uint32) << 16).view(np.float32)
    return out[:, 0], out[:, 1]


def decode_T(T, n_tiles, Ci, F, P):
    """tile layout [tile][ifb][4][PH][128][4] -> [n_tiles*128, Ci*F, P]."""
    nifb = (Ci * F + 3) // 4
    ph = (P + 3) // 4
    t = T[: n_tiles * nifb * 4 * ph * 128 * 4].reshape(n_tiles, nifb * 4, ph, 128, 4)
    t = t.transpose(0, 3, 1, 2, 4).reshape(n_tiles * 128, nifb * 4, ph * 4)
    return t[:, : Ci * F, :P]
