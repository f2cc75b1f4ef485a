"""Peak device memory and time of forwards whose edge work runs over node chunks under the edge budget (SE3B200_EDGE_BUDGET_MB,
DESIGN.md 4.7).  Workloads:

  headline16k_default / headline16k_8gb   the headline model (dim 512, 8 heads of 64, depth 6, 4 degrees, k = 16) on 1 x 16 384
                                          points, at the default budget and at 8 GB
  headline50k / headline100k             the same model on 1 x 50 000 and 1 x 100 000 points (default budget)
  allnbr2048 / allnbr4096                dim 128, 2 heads of 64, depth 1, 4 degrees, output_degrees 2, num_neighbors = inf on
                                          2049 and 4097 points (k = 2048 and 4096), 8 GB budget

For each: median ms per forward over --steps timed forwards after --warmup, us per edge, the peak of
torch.cuda.max_memory_allocated over one forward above what was allocated before it (the resident weights of both models and the
inputs, also reported), and the node chunks run (all blocks, and the most in one block).  Prints one JSON
line with the card's name and power limit (read-only nvidia-smi query).  Writes nothing.

    python bench_memory.py [--steps 1] [--warmup 1] [--only headline16k_default,allnbr2048]
"""
import argparse
import json

import numpy as np
import torch

from bench_varlen import card

HEADLINE = dict(dim=512, heads=8, dim_head=64, depth=6, num_degrees=4, num_neighbors=16)
ALLNBR = dict(dim=128, heads=2, dim_head=64, depth=1, num_degrees=4, output_degrees=2, num_neighbors=float('inf'))
WORKLOADS = {                        # name: (model, points, edge budget in MiB or None for the default)
    'headline16k_default': ('headline', 16384, None),
    'headline16k_8gb': ('headline', 16384, 8192),
    'headline50k': ('headline', 50000, None),
    'headline100k': ('headline', 100000, None),
    'allnbr2048': ('allnbr', 2049, 8192),
    'allnbr4096': ('allnbr', 4097, 8192),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=1)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--only', default=','.join(WORKLOADS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_memory.py measures on a CUDA device; none found')
    from se3_transformer_pytorch_b200 import SE3Transformer, model as M, switches

    dev = torch.device('cuda')
    models = {}
    torch.manual_seed(1234)
    with torch.device(dev):
        models['headline'] = SE3Transformer(**HEADLINE).eval()
        models['allnbr'] = SE3Transformer(**ALLNBR).eval()
    models['headline'].pack_weights(free_master=True, max_distance=16.0)     # as bench.py

    plans, orig = [], M.plan_node_chunks

    def recording(*a):
        chunks = orig(*a)
        plans.append(len(chunks))
        return chunks
    M.plan_node_chunks = recording

    gpu, power = card()
    res = dict(workload='edge_budget_memory', steps=args.steps, warmup=args.warmup, gpu=gpu, power_limit=power,
               default_budget_gb=round(M.edge_budget_bytes(switches.current(), dev) / 1e9, 2))
    g = torch.Generator().manual_seed(99)
    for name in args.only.split(','):
        which, n, budget = WORKLOADS[name]
        model = models[which]
        feats = torch.randn(1, n, model.dim, generator=g).to(dev)
        coors = (torch.randn(1, n, 3, generator=g) * (3.0 if which == 'allnbr' else 1.0)).to(dev)
        k = int(min(model.num_neighbors, n - 1))
        times, peak, resident = [], 0, torch.cuda.memory_allocated()
        with torch.no_grad(), switches.override(edge_budget_mb=budget):
            for step in range(args.warmup + args.steps):
                del plans[:]
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = model(feats, coors)
                e1.record()
                torch.cuda.synchronize()
                peak = max(peak, torch.cuda.max_memory_allocated() - resident)
                if step >= args.warmup:
                    times.append(e0.elapsed_time(e1))
                del out
        ms = float(np.median(times))
        res[name] = dict(n=n, k=k, edges=n * k, budget_mb=budget, ms=round(ms, 1), us_per_edge=round(ms * 1e3 / (n * k), 3),
                         peak_gb=round(peak / 1e9, 2), resident_gb=round(resident / 1e9, 2), chunks=sum(plans), blocks=len(plans),
                         max_chunks_per_block=max(plans))
        print(json.dumps({name: res[name]}), flush=True)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
