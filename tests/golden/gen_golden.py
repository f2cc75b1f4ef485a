"""Golden-vector generator.  Needs a checkout of the real reference (lucidrains/se3-transformer-pytorch) on the Python path
and writes small fixtures that travel with the repo; the tests themselves never import the reference.

    PYTHONPATH=<reference checkout> CACHE_PATH=/tmp/se3_cache python tests/golden/gen_golden.py

Outputs
  se3_transformer_pytorch_b200/data/qj_tables.npz   Q_J change-of-basis tables (reference basis.py:123-138)
  tests/golden/sh_basis.npz                         Y_J + get_basis on fixed vectors (basis.py:140-205)
  tests/golden/model_<case>.npz                     whole-model inputs/outputs + captured intermediates (largest arrays
                                                    in model_<case>.part<i>.npz, so that every file stays under 1 MB)
  tests/golden/state_keys.json                      state_dict key/shape lists (SURVEY.md A.6); the DEG_CASES fixtures
                                                    hold their own as 'state_keys'

Weights are never stored: both sides fill state_dict() with tests/golden/detfill.py.
"""
import os, sys, json
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
os.environ.setdefault('CACHE_PATH', '/tmp/se3_cache')

from detfill import fill_state_dict, det_inputs, det_uniform  # noqa: E402
import se3_transformer_pytorch.se3_transformer_pytorch as ref_mod  # noqa: E402
from se3_transformer_pytorch.basis import basis_transformation_Q_J, get_basis, get_spherical_from_cartesian, precompute_sh  # noqa: E402
from se3_transformer_pytorch.irr_repr import rot  # noqa: E402

MAX_TABLE_DEGREE = 5


def gen_qj():
    out = {}
    for lo in range(MAX_TABLE_DEGREE + 1):
        for li in range(MAX_TABLE_DEGREE + 1):
            for J in range(abs(li - lo), li + lo + 1):
                out[f'{J}_{li}_{lo}'] = basis_transformation_Q_J(J, li, lo).numpy().astype(np.float32)
    path = os.path.join(ROOT, 'se3_transformer_pytorch_b200', 'data', 'qj_tables.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, len(out), 'tables')


def special_vectors():
    v = det_inputs('sh_vectors', (56, 3), seed=3)
    extra = np.array([
        [0, 0, 0], [0, 1, 0], [0, -1, 0], [1, 0, 0], [0, 0, 1], [-1, 0, 0], [0, 0, -1], [1e-4, 2.0, -1e-4],
    ], dtype=np.float32)
    return np.concatenate([v, extra], 0)


def gen_sh_basis():
    r = torch.from_numpy(special_vectors())
    out = {'r_ij': r.numpy()}
    sph = get_spherical_from_cartesian(r.clone())
    Y = precompute_sh(sph, 6)
    for J, y in Y.items():
        out[f'Y_{J}'] = y.numpy()
    basis = get_basis(r.clone(), 3)
    for k, v in basis.items():
        li, lo = map(int, k.split(','))
        out[f'basis_{li}_{lo}'] = v.reshape(r.shape[0], 2 * lo + 1, 2 * li + 1, 2 * min(li, lo) + 1).numpy()
    # fp64 reference as well (tighter oracle pin)
    r64 = r.double()
    sph64 = get_spherical_from_cartesian(r64.clone())
    Y64 = precompute_sh(sph64, 6)
    for J, y in Y64.items():
        out[f'Y64_{J}'] = y.numpy()
    path = os.path.join(HERE, 'sh_basis.npz')
    np.savez_compressed(path, **out)
    print('wrote', path)


def band_adj(n, w):
    i = np.arange(n)
    return (np.abs(i[:, None] - i[None, :]) <= w) & (i[:, None] != i[None, :])


CASES = [
    dict(name='cfg1', ctor=dict(dim=64, depth=2, num_degrees=2, num_neighbors=8), b=1, n=32, capture_kv=True),
    dict(name='deg4', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=4, output_degrees=2, num_neighbors=6, valid_radius=10),
         b=2, n=24, capture_kv=True),
    dict(name='af2', ctor=dict(dim=32, heads=4, dim_head=8, depth=2, input_degrees=1, num_degrees=2, output_degrees=2, reduce_dim_out=True,
                               num_neighbors=8), b=2, n=48, fwd=dict(return_type=1)),
    dict(name='edges_sparse', ctor=dict(dim=32, heads=4, dim_head=8, depth=1, num_degrees=3, num_edge_tokens=4, edge_dim=8,
                                        attend_sparse_neighbors=True, num_neighbors=0, max_sparse_neighbors=8),
         b=2, n=32, edges='tokens', adj=4),
    dict(name='ragged', ctor=dict(dim=16, dim_in=(16, 4), heads=2, dim_head=8, depth=1, input_degrees=2, num_degrees=3, output_degrees=2,
                                  num_neighbors=5, valid_radius=1.5, fourier_encode_dist=True),
         b=2, n=20, ragged=True, type1_in=True),
    dict(name='tc_deg2', ctor=dict(dim=32, heads=2, dim_head=16, depth=1, num_degrees=2, output_degrees=2, num_neighbors=8), b=2, n=64,
         capture_kv=True),
    dict(name='tc_deg4', ctor=dict(dim=32, heads=2, dim_head=16, depth=1, num_degrees=4, num_neighbors=4), b=2, n=32),
    dict(name='allnbr', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2), b=1, n=12),
    dict(name='causal', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=4, causal=True), b=1, n=16),
    dict(name='tiekv', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=4, tie_key_values=True), b=1, n=16),
    dict(name='linkeys', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=4, linear_proj_keys=True), b=1, n=16),
    dict(name='nullkv', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=4, use_null_kv=True), b=1, n=16),
    dict(name='noself', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=4, attend_self=False), b=1, n=16),
    dict(name='global', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=4, global_feats_dim=8), b=1, n=16,
         global_feats=(3, 8)),
    dict(name='onehead', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=4, one_headed_key_values=True), b=1, n=16),
    dict(name='preconv_normout', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, output_degrees=2, num_neighbors=4,
                                           num_conv_layers=1, norm_out=True), b=1, n=16, fwd=dict(return_pooled=True)),
    dict(name='tokens_pos', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=4, num_tokens=7, num_positions=32),
         b=2, n=16, tokens=7),
    dict(name='adjdeg', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=3, attend_sparse_neighbors=True,
                                  num_adj_degrees=2, adj_dim=4), b=1, n=16, adj=1),
    dict(name='nbrmask', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=4, valid_radius=10), b=1, n=16,
         neighbor_mask=True),
    dict(name='contedges', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, output_degrees=2, edge_dim=6, num_neighbors=5),
         b=2, n=12, edges='continuous', fwd=dict(return_type=1)),
]


# BASELINE.json configs[2] at full size and configs[3] at batch 2 (outputs only; ~20 s and ~5 min of reference CPU time)
BIG_CASES = [
    dict(name='cfg3', ctor=dict(dim=64, depth=2, input_degrees=1, num_degrees=2, output_degrees=2, reduce_dim_out=True, num_neighbors=16),
         b=2, n=256, fwd=dict(return_type=1), no_capture=True),
    # configs[3] with batch 2 instead of 8: the reference needs ~8 GB per cloud here (band adjacency, 8 bonded neighbours)
    dict(name='cfg4_b2', ctor=dict(dim=128, depth=2, num_degrees=3, num_edge_tokens=4, edge_dim=16, attend_sparse_neighbors=True,
                                   num_neighbors=0, max_sparse_neighbors=8), b=2, n=512, edges='tokens', adj=4, no_capture=True),
]


# widths the one-GEMM production kernel takes (every fiber a multiple of 128 channels; DESIGN.md 4.5), small enough for the
# reference's materialising CPU path
ZCASES = [
    dict(name='z128', ctor=dict(dim=128, heads=2, dim_head=64, depth=1, num_degrees=3, output_degrees=2, num_neighbors=6, valid_radius=10),
         b=1, n=20, no_capture=True),
    dict(name='z256_deg4', ctor=dict(dim=256, heads=4, dim_head=64, depth=1, num_degrees=4, num_neighbors=5), b=2, n=14, no_capture=True),
]


# rotary embeddings (reference rotary.py, S:488-494, 1298-1325; tests/test_equivariance.py:184-203)
RCASES = [
    dict(name='rotary_both', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, attend_self=True, num_neighbors=4, num_degrees=2, output_degrees=2,
                                       fourier_encode_dist=True, rotary_position=True, rotary_rel_dist=True), b=2, n=16),
    dict(name='rotary_pos_onehead', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_neighbors=4, num_degrees=2, rotary_position=True,
                                              one_headed_key_values=True, use_null_kv=True), b=1, n=16),
    dict(name='rotary_dist_linkeys', ctor=dict(dim=16, heads=2, dim_head=8, depth=2, num_neighbors=5, num_degrees=3, rotary_rel_dist=True,
                                               linear_proj_keys=True), b=1, n=12),
    dict(name='rotary_tiekv', ctor=dict(dim=16, heads=2, dim_head=12, depth=1, num_neighbors=4, num_degrees=2, rotary_position=True,
                                        rotary_rel_dist=True, tie_key_values=True), b=1, n=12),
]


# the top of the documented degree range (num_degrees 5 and 6: Q_J tables and kernel templates up to degree 5).  tc_deg5 puts
# the tensor-core kernels on pairs with degree_in = 4 and SIMT on degree_out = 4; z128_deg6 runs the attention convolutions on
# the mixed low-rank / SIMT route and conv_out (outputs of degree <= 1) on the one-GEMM path with inputs up to degree 5.
# These models have ~1000 parameter tensors each: their state_dict layout is stored in the fixture ('state_keys'), not in
# state_keys.json.
DEG_CASES = [
    dict(name='deg6', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=6, output_degrees=2, num_neighbors=4), b=1, n=10,
         capture_kv=True),
    dict(name='tc_deg5', ctor=dict(dim=32, heads=2, dim_head=16, depth=1, num_degrees=5, output_degrees=2, num_neighbors=6), b=1, n=16),
    dict(name='z128_deg6', ctor=dict(dim=128, heads=2, dim_head=64, depth=1, num_degrees=6, output_degrees=2, num_neighbors=4), b=1, n=8,
         no_capture=True),
]


def build_inputs(case):
    b, n = case['b'], case['n']
    name = case['name']
    ctor = case['ctor']
    inp = {}
    dim_in = ctor.get('dim_in', ctor['dim'])
    if case.get('tokens'):
        u = det_uniform('tok/' + name, b * n, 1)
        inp['feats'] = (u * case['tokens']).astype(np.int64).reshape(b, n)
    elif case.get('type1_in'):
        inp['feats/0'] = det_inputs(name + '/f0', (b, n, dim_in[0], 1), 1)
        inp['feats/1'] = det_inputs(name + '/f1', (b, n, dim_in[1], 3), 1)
    else:
        inp['feats'] = det_inputs(name + '/feats', (b, n, dim_in), 1)
    inp['coors'] = det_inputs(name + '/coors', (b, n, 3), 2)
    mask = np.ones((b, n), dtype=bool)
    if case.get('ragged'):
        for bi in range(b):
            mask[bi, n - 3 * (bi + 1):] = False
    inp['mask'] = mask
    if case.get('adj') is not None:
        inp['adj_mat'] = band_adj(n, case['adj'])
    if case.get('edges') == 'tokens':
        u = det_uniform('edge/' + name, b * n * n, 1)
        inp['edges'] = (u * ctor['num_edge_tokens']).astype(np.int64).reshape(b, n, n)
    elif case.get('edges') == 'continuous':
        inp['edges'] = det_inputs(name + '/edges', (b, n, n, ctor['edge_dim']), 5)
    if case.get('neighbor_mask'):
        u = det_uniform('nm/' + name, b * n * n, 1).reshape(b, n, n)
        inp['neighbor_mask'] = u < 0.6
    if case.get('global_feats'):
        g, d = case['global_feats']
        inp['global_feats'] = det_inputs(name + '/global', (b, g, d), 4)
    return inp


def to_np(t):
    return t.detach().cpu().numpy()


def run_case(case):
    name = case['name']
    torch.manual_seed(0)
    model = ref_mod.SE3Transformer(**case['ctor'])
    fill_state_dict(model, seed=11)
    model.eval()
    inp = build_inputs(case)
    out = dict(('in/' + k, v) for k, v in inp.items())

    cap = {}
    orig_get_basis = ref_mod.get_basis

    def patched_get_basis(r_ij, max_degree, differentiable=False):
        cap['graph/rel_pos'] = to_np(r_ij)
        return orig_get_basis(r_ij, max_degree, differentiable=differentiable)

    ref_mod.get_basis = patched_get_basis
    hooks = []

    def conv_in_pre(mod, args, kwargs):
        x, edge_info = args[0], args[1]
        idx, nmask, edges = edge_info
        cap['graph/neighbor_indices'] = to_np(idx)
        cap['graph/neighbor_mask'] = to_np(nmask)
        if edges is not None:
            cap['graph/edges'] = to_np(edges)
        cap['graph/rel_dist'] = to_np(kwargs['rel_dist'])
        for d, t in x.items():
            cap[f'conv_in/in/{d}'] = to_np(t)

    def conv_in_post(mod, args, kwargs, output):
        for d, t in output.items():
            cap[f'conv_in/out/{d}'] = to_np(t)

    if not case.get('no_capture'):
        hooks.append(model.conv_in.register_forward_pre_hook(conv_in_pre, with_kwargs=True))
        hooks.append(model.conv_in.register_forward_hook(conv_in_post, with_kwargs=True))

    if not case['ctor'].get('use_egnn') and not case.get('no_capture'):
        attn = model.net.blocks[0][0].attn

        def attn_pre(mod, args, kwargs):
            for d, t in args[0].items():
                cap[f'attn0/in/{d}'] = to_np(t)

        def attn_post(mod, args, kwargs, output):
            for d, t in output.items():
                cap[f'attn0/out/{d}'] = to_np(t)

        hooks.append(attn.register_forward_pre_hook(attn_pre, with_kwargs=True))
        hooks.append(attn.register_forward_hook(attn_post, with_kwargs=True))
        if case.get('capture_kv'):
            def mk(tag):
                def h(mod, args, kwargs, output):
                    for d, t in output.items():
                        cap[f'attn0/{tag}/{d}'] = to_np(t)
                return h
            hooks.append(attn.to_v.register_forward_hook(mk('v'), with_kwargs=True))
            if getattr(attn, 'to_k', None) is not None and isinstance(attn.to_k, ref_mod.ConvSE3):
                hooks.append(attn.to_k.register_forward_hook(mk('k'), with_kwargs=True))

    # forward
    if 'feats' in inp:
        feats = torch.from_numpy(inp['feats'])
    else:
        feats = {'0': torch.from_numpy(inp['feats/0']), '1': torch.from_numpy(inp['feats/1'])}
    kwargs = dict(case.get('fwd', {}))
    for k in ('adj_mat', 'edges', 'neighbor_mask', 'global_feats'):
        if k in inp:
            kwargs[k] = torch.from_numpy(inp[k])
    with torch.no_grad():
        res = model(feats, torch.from_numpy(inp['coors']), torch.from_numpy(inp['mask']), **kwargs)
    ref_mod.get_basis = orig_get_basis
    for h in hooks:
        h.remove()

    if torch.is_tensor(res):
        out['out'] = to_np(res)
    else:
        for d, t in res.items():
            out[f'out/{d}'] = to_np(t)
    for k, v in cap.items():
        out['cap/' + k] = v
    out['config'] = np.array(json.dumps(dict(ctor={k: (list(v) if isinstance(v, tuple) else v) for k, v in case['ctor'].items()},
                                             fwd=case.get('fwd', {}), b=case['b'], n=case['n'])))
    keys = {k: list(v.shape) for k, v in model.state_dict().items()}
    if name in {c['name'] for c in DEG_CASES}:
        out['state_keys'] = np.array(json.dumps(keys, sort_keys=True))
    path = os.path.join(HERE, f'model_{name}.npz')
    write_split(path, out)
    print('wrote', path, 'params', sum(int(np.prod(s)) for s in keys.values()), 'size', os.path.getsize(path))
    return keys


def write_split(path, arrays, limit=900_000):
    """np.savez_compressed(path, **arrays), moving the largest arrays one by one into path.part<i>.npz files while a file
    would exceed `limit` bytes (tests/helpers.py:load_case merges them back)."""
    import io
    for old in [f for f in os.listdir(HERE) if f.startswith(os.path.basename(path)[:-4] + '.part')]:
        os.remove(os.path.join(HERE, old))
    main = dict(arrays)
    size = lambda d: (lambda b: (np.savez_compressed(b, **d), b.tell())[1])(io.BytesIO())
    parts = []
    for k in sorted(main, key=lambda k: -main[k].nbytes):
        if size(main) <= limit:
            break
        if k in ('config', 'state_keys'):
            continue
        if parts and size({**parts[-1], k: main[k]}) <= limit:
            parts[-1][k] = main.pop(k)
        else:
            parts.append({k: main.pop(k)})
    np.savez_compressed(path, **main)
    for i, part in enumerate(parts):
        np.savez_compressed(f'{path[:-4]}.part{i + 2}.npz', **part)


def gen_equivariance_inputs():
    """The rotation used by the reference's own equivariance tests (tests/test_equivariance.py:158)."""
    R = rot(15, 0, 45).numpy()
    np.savez(os.path.join(HERE, 'rot_15_0_45.npz'), R=R)


if __name__ == '__main__':
    which = sys.argv[1:] or ['qj', 'sh', 'models', 'rot']
    if 'qj' in which:
        gen_qj()
    if 'sh' in which:
        gen_sh_basis()
    if 'rot' in which:
        gen_equivariance_inputs()
    if 'deg' in which:
        for case in DEG_CASES:
            run_case(case)
    if 'models' in which or 'big' in which or 'z' in which or 'rotary' in which:
        kpath = os.path.join(HERE, 'state_keys.json')
        all_keys = json.load(open(kpath)) if os.path.exists(kpath) else {}
        for case in (CASES if 'models' in which else []) + (BIG_CASES if 'big' in which else []) + (ZCASES if 'z' in which else []) + (RCASES if 'rotary' in which else []):
            all_keys[case['name']] = run_case(case)
        with open(kpath, 'w') as f:
            json.dump(all_keys, f, indent=0, sort_keys=True)
