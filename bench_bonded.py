"""Bonded clouds with sparse pair inputs: the model of the 10k dense-pair-input test (bonded chains, their 2-hop adjacency as
hop-count embeddings, edge tokens, neighbor_mask; dim 16, 8 local + bonded neighbours) on clouds made of parts of ~3400 points
1e4 apart.  Within a part, node i is bonded to i +- 1, carries an edge token in 1..3 to every node within 32 positions (token 0
elsewhere), and its neighbor_mask allows a random 70 % of those 64 nodes.  So the pair data is O(n), as for a molecule.

At n = 10 200 (3 parts) the forward runs on the dense [n, n] pair inputs (the reference's format) and on the same inputs as
torch.sparse_coo tensors, alternating; at n = 50 000 (15 parts) and 100 000 (30 parts) on the sparse inputs only.  For each, after
a warm-up, the forward is timed with CUDA events over --steps steps, its peak device memory above what was allocated before the
call (inputs and weights) is read from torch's allocator, and one more profiled forward gives the time of the `knn` kernel
(the neighbour search, O(n^2) work).  Prints one JSON line, with the card's name and power limit (read-only nvidia-smi query).

    python bench_bonded.py [--steps 3] [--warmup 1] [--sizes 10200,50000,100000]
"""
import argparse
import contextlib
import json
import sys

import numpy as np
import torch

from bench_varlen import card

CTOR = dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, output_degrees=2, num_neighbors=8, attend_sparse_neighbors=True,
            max_sparse_neighbors=8, num_adj_degrees=2, adj_dim=4, num_edge_tokens=4, edge_dim=4)
PART = 3400                                # nodes per part, at most
WINDOW = 32                                # edge tokens and neighbor_mask candidates: nodes within this many positions


def bonded_parts(n, parts, device, seed=0):
    """feats [1, n, 16], coors [1, n, 3] and sparse adj_mat [n, n] bool, edges [1, n, n] int64, neighbor_mask [1, n, n] bool of
    `parts` parts 1e4 apart (node i in part i * parts // n), and the parts' (start, end)."""
    g = torch.Generator(device=device).manual_seed(seed)
    i = torch.arange(n, device=device)
    part = i * parts // n
    coors = torch.randn(n, 3, generator=g, device=device) * 10
    coors[:, 0] += part * 1e4
    feats = torch.randn(1, n, CTOR['dim'], generator=g, device=device)
    off = torch.cat((torch.arange(-WINDOW, 0), torch.arange(1, WINDOW + 1))).to(device)
    r = i.repeat_interleave(off.numel())
    c = r + off.repeat(n)
    ok = (c >= 0) & (c < n)
    r, c = r[ok], c[ok]
    ok = part[r] == part[c]
    r, c = r[ok], c[ok]
    z = torch.zeros_like(r)
    bond = (r - c).abs() == 1
    adj = torch.sparse_coo_tensor(torch.stack((r[bond], c[bond])), torch.ones(int(bond.sum()), dtype=torch.bool, device=device), (n, n))
    keep = torch.rand(r.numel(), generator=g, device=device) < 0.7
    nbr = torch.sparse_coo_tensor(torch.stack((z[keep], r[keep], c[keep])), torch.ones(int(keep.sum()), dtype=torch.bool, device=device),
                                  (1, n, n))
    tokens = torch.randint(1, 4, (r.numel(),), generator=g, device=device)
    edges = torch.sparse_coo_tensor(torch.stack((z, r, c)), tokens, (1, n, n))
    ends = torch.bincount(part, minlength=parts).cumsum(0).tolist()
    return feats, coors[None], adj, edges, nbr, list(zip([0] + ends[:-1], ends))


def measure(model, feats, coors, kw):
    """(forward ms, peak bytes above the memory allocated before the call)"""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    model(feats, coors, **kw)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), torch.cuda.max_memory_allocated() - base


def knn_ms(model, feats, coors, kw):
    """Time of the knn kernel in one profiled forward (CUDA events around the launch)."""
    from se3_transformer_pytorch_b200 import ops
    ops.PROFILE = []
    try:
        model(feats, coors, **kw)
        torch.cuda.synchronize()
        return sum(p[1].elapsed_time(p[2]) for p in ops.PROFILE if p[0] == 'knn')
    finally:
        ops.PROFILE = None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--sizes', default='10200,50000,100000')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_bonded.py measures on a CUDA device; none found')
    with contextlib.redirect_stdout(sys.stderr):      # forward prints the reference's neighbor_mask notice; stdout is the JSON line
        res = run(args)
    print(json.dumps(res))


def run(args):
    from se3_transformer_pytorch_b200 import SE3Transformer

    dev = torch.device('cuda')
    torch.manual_seed(1234)
    model = SE3Transformer(**CTOR).to(dev).eval()
    runs = {}
    for n in [int(s) for s in args.sizes.split(',')]:
        parts = -(-n // PART)
        feats, coors, adj, edges, nbr, _ = bonded_parts(n, parts, dev, seed=n)
        sparse = dict(adj_mat=adj, edges=edges, neighbor_mask=nbr)
        nnz = {k: int(v._nnz()) for k, v in sparse.items()}
        if n <= 16384:                          # the dense inputs of larger clouds take O(n^2) memory: 80 GB of edges at 10^5
            runs[f'n{n}_dense'] = (n, parts, nnz, feats, coors, {k: v.to_dense() for k, v in sparse.items()})
        runs[f'n{n}_sparse'] = (n, parts, nnz, feats, coors, sparse)

    times = {name: [] for name in runs}
    peaks = {name: 0 for name in runs}
    for step in range(args.warmup + args.steps):
        for name, (_, _, _, feats, coors, kw) in runs.items():       # dense and sparse alternate
            ms, peak = measure(model, feats, coors, kw)
            peaks[name] = max(peaks[name], peak)
            if step >= args.warmup:
                times[name].append(ms)

    gpu, power = card()
    res = dict(workload='bonded_sparse_pairs', ctor=CTOR, part=PART, window=WINDOW, steps=args.steps, warmup=args.warmup, gpu=gpu,
               power_limit=power)
    for name, (n, parts, nnz, feats, coors, kw) in runs.items():
        ms = float(np.median(times[name]))
        row = dict(n=n, parts=parts, nnz=nnz, ms_median=round(ms, 2), ms_min=round(float(min(times[name])), 2),
                   ms_max=round(float(max(times[name])), 2), peak_mb=round(peaks[name] / 2 ** 20, 1),
                   pair_input_mb=round(sum(t.numel() * t.element_size() if not t.is_sparse else
                                           t._indices().numel() * 8 + t._values().numel() * t._values().element_size()
                                           for t in kw.values()) / 2 ** 20, 1),
                   knn_ms=round(knn_ms(model, feats, coors, kw), 3))
        row['knn_share'] = round(row['knn_ms'] / ms, 4)
        res[name] = row
    return res


if __name__ == '__main__':
    main()
