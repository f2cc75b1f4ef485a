"""Padded against packed: the headline model (dim 512, 8 heads of 64, depth 6, 4 degrees, k = 16) on a protein-like batch of
clouds of 1024, 832, 640 and 448 nodes.

  (a) forward():        padded to [4, 1024] with a node mask; the padding nodes sit 1e4 away from every real node, so no real
                        node gives a neighbour slot to them and the real nodes' outputs equal the packed ones;
  (b) forward_packed(): the clouds concatenated, T = 2944 nodes.

Both run in one process, alternating step by step, each step timed with CUDA events after a warm-up.  Prints one JSON line: ms
per forward, clouds/s, edges built, the per-cloud relative difference of (a) and (b) on the real nodes, and the card's name and
power limit (read-only nvidia-smi query).  The edge counts are arithmetic; the times are what this card measured.

    python bench_varlen.py [--steps 10] [--warmup 2]
"""
import argparse
import json
import subprocess

import numpy as np
import torch

LENS = [1024, 832, 640, 448]
CTOR = dict(dim=512, heads=8, dim_head=64, depth=6, num_degrees=4, num_neighbors=16)


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, power = (s.strip() for s in out[torch.cuda.current_device()].split(','))
        return name, power
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(), 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_varlen.py measures on a CUDA device; none found')
    from se3_transformer_pytorch_b200 import SE3Transformer

    dev = torch.device('cuda')
    torch.manual_seed(1234)
    with torch.device(dev):
        model = SE3Transformer(**CTOR).eval()
    model.pack_weights(free_master=True, max_distance=16.0)         # as bench.py: low-rank plan for distances <= 16, masters released
    B, n_max, T, dim, k = len(LENS), max(LENS), sum(LENS), CTOR['dim'], CTOR['num_neighbors']
    g = torch.Generator().manual_seed(99)
    feats = torch.randn(T, dim, generator=g)
    coors = torch.randn(T, 3, generator=g)
    # padded batch: padding features zero, padding coordinates 1e4 away from the real ones (and close to each other)
    p_feats = torch.zeros(B, n_max, dim)
    p_coors = torch.randn(B, n_max, 3, generator=g) + torch.tensor([1e4, 0., 0.])
    p_mask = torch.zeros(B, n_max, dtype=torch.bool)
    s = 0
    for c, n in enumerate(LENS):
        p_feats[c, :n], p_coors[c, :n], p_mask[c, :n] = feats[s:s + n], coors[s:s + n], True
        s += n
    feats, coors, p_feats, p_coors, p_mask = (t.to(dev) for t in (feats, coors, p_feats, p_coors, p_mask))

    runs = {'padded': lambda: model(p_feats, p_coors, p_mask), 'packed': lambda: model.forward_packed(feats, coors, LENS)}
    times = {name: [] for name in runs}
    out = {}
    for step in range(args.warmup + args.steps):
        for name, fn in runs.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out[name] = fn()
            e1.record()
            torch.cuda.synchronize()
            if step >= args.warmup:
                times[name].append(e0.elapsed_time(e1))

    errs, s = [], 0
    for c, n in enumerate(LENS):
        a = out['padded'][c, :n].double().cpu().numpy()
        b = out['packed'][s:s + n].double().cpu().numpy()
        errs.append(float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)))
        s += n
    name, power = card()
    res = dict(workload='varlen_headline', lens=LENS, ctor=CTOR, steps=args.steps, warmup=args.warmup, gpu=name, power_limit=power)
    edges = {'padded': B * n_max * k, 'packed': T * k}
    for key, ts in times.items():
        ms = float(np.median(ts))
        res[key] = dict(ms_median=round(ms, 2), ms_min=round(float(min(ts)), 2), ms_max=round(float(max(ts)), 2),
                        clouds_per_s=round(B / (ms / 1e3), 3), edges=edges[key])
    res['edge_ratio'] = round(edges['packed'] / edges['padded'], 4)
    res['speedup'] = round(res['padded']['ms_median'] / res['packed']['ms_median'], 3)
    res['rel_err_padded_vs_packed'] = [float(f'{e:.3e}') for e in errs]
    print(json.dumps(res))


if __name__ == '__main__':
    main()
