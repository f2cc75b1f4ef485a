"""One large cloud through forward(): the headline model (dim 512, 8 heads of 64, depth 6, 4 degrees, k = 16) on a single cloud
of n = 4097 (the longest row the neighbour search sorts whole), 8192 and 16384 points (rows searched in tiles of 4096 columns).
bench.py's workload (4 clouds of 1024 points) runs alongside with the same weights, so that the per-edge times sit side by side.

For every size, after a warm-up, the forward is timed with CUDA events over --steps steps, alternating between the sizes.  One
more profiled forward per size gives the time of the `knn` kernel.  The cloud is also split into two halves 1e4 apart (the second
half moved away); with k = 16 no neighbour crosses between them, so the output must equal forward() on each half alone, and the
largest relative difference is reported.  Prints one JSON line, with the card's name and power limit (read-only nvidia-smi query).

    python bench_large.py [--steps 3] [--warmup 1] [--sizes 4097,8192,16384]
"""
import argparse
import json

import numpy as np
import torch

from bench_varlen import card

CTOR = dict(dim=512, heads=8, dim_head=64, depth=6, num_degrees=4, num_neighbors=16)
BENCH_WORKLOAD = (4, 1024)                 # bench.py's cfg2: b clouds of n points


def knn_ms(model, feats, coors):
    """Time of the knn kernel in one profiled forward (CUDA events around the launch)."""
    from se3_transformer_pytorch_b200 import ops
    ops.PROFILE = []
    try:
        model(feats, coors)
        torch.cuda.synchronize()
        return sum(p[1].elapsed_time(p[2]) for p in ops.PROFILE if p[0] == 'knn')
    finally:
        ops.PROFILE = None


def halves_rel_err(model, feats, coors, out):
    """Largest relative difference between the whole cloud's output and forward() on each half alone (0.0: bit-identical)."""
    n = coors.shape[1]
    as_dict = lambda o: o if isinstance(o, dict) else {'0': o}
    errs = []
    for s, e in ((0, n // 2), (n // 2, n)):
        part = as_dict(model(feats[:, s:e].contiguous(), coors[:, s:e].contiguous()))
        for d, whole in as_dict(out).items():
            a, b = whole[:, s:e].double(), part[d].double()
            errs.append(float((a - b).abs().max() / b.abs().max().clamp_min(1e-30)))
    return max(errs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--sizes', default='4097,8192,16384')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_large.py measures on a CUDA device; none found')
    from se3_transformer_pytorch_b200 import SE3Transformer

    dev = torch.device('cuda')
    torch.manual_seed(1234)
    with torch.device(dev):
        model = SE3Transformer(**CTOR).eval()
    model.pack_weights(free_master=True, max_distance=16.0)         # as bench.py: low-rank plan for distances <= 16, masters released
    g = torch.Generator().manual_seed(99)
    inputs = {}
    for n in [int(s) for s in args.sizes.split(',')]:
        coors = torch.randn(1, n, 3, generator=g)
        coors[:, n // 2:, 0] += 1e4                                 # two halves 1e4 apart
        inputs[f'n{n}'] = (1, n, torch.randn(1, n, CTOR['dim'], generator=g).to(dev), coors.to(dev))
    b, n = BENCH_WORKLOAD
    inputs['bench_py'] = (b, n, torch.randn(b, n, CTOR['dim'], generator=g).to(dev), torch.randn(b, n, 3, generator=g).to(dev))

    times = {name: [] for name in inputs}
    out = {}
    for step in range(args.warmup + args.steps):
        for name, (_, _, feats, coors) in inputs.items():
            out.pop(name, None)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            res = model(feats, coors)
            e1.record()
            torch.cuda.synchronize()
            if step >= args.warmup:
                times[name].append(e0.elapsed_time(e1))
            if step == args.warmup + args.steps - 1:
                out[name] = res

    gpu, power = card()
    res = dict(workload='large_cloud_headline', ctor=CTOR, steps=args.steps, warmup=args.warmup, gpu=gpu, power_limit=power)
    for name, (b, n, feats, coors) in inputs.items():
        ms = float(np.median(times[name]))
        edges = b * n * CTOR['num_neighbors']
        row = dict(clouds=b, n=n, edges=edges, ms_median=round(ms, 2), ms_min=round(float(min(times[name])), 2),
                   ms_max=round(float(max(times[name])), 2), ms_per_cloud=round(ms / b, 2), us_per_edge=round(ms * 1e3 / edges, 3),
                   knn_ms=round(knn_ms(model, feats, coors), 3))
        row['knn_share'] = round(row['knn_ms'] / ms, 5)
        if b == 1:
            row['halves_max_rel_err'] = halves_rel_err(model, feats, coors, out[name])
        res[name] = row
    print(json.dumps(res))


if __name__ == '__main__':
    main()
