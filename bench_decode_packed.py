"""Continuous batching with the packed causal decoder against one decoder per request and static lockstep batches, on a trace
of requests with prompts and generation lengths of different sizes, with bench_decode.py's model (the README's autoregressive
model: dim 512, 8 x 64 heads, depth 6, 4 degrees, valid_radius 10, causal, k = 16), weights and production path.

    python bench_decode_packed.py [--requests 32] [--reps 2] [--slots 4 16]

Trace (seeded): prompt lengths spread over [256, 960], 16 .. 64 generated single nodes each, coordinates N(0, 9) as in
bench_decode.py.  Schedules, each run once to warm every step shape and then --reps times timed:
  (a) PackedCausalDecoder with at most S clouds in flight: a waiting request joins as soon as a cloud closes, its prompt riding in
      the same step as the other clouds' single nodes;
  (b) one batch-1 CausalDecoder per request, in sequence;
  (c) static lockstep batches of S requests: prompts left-padded with masked nodes, every cloud stepping until the batch's
      longest request finishes (exact for this model, which has no positions).
Every step ends in a device synchronise.  Prints one line per run and a JSON summary with the card and its power limit."""
import argparse
import json
import sys
import time

import numpy as np
import torch

from bench_decode import CTOR, card, fill_device


def trace(requests, seed=0):
    rng = np.random.default_rng(seed)
    prompts = rng.integers(256, 961, requests).tolist()
    gens = rng.integers(16, 65, requests).tolist()
    g = torch.Generator().manual_seed(seed)
    data = [(torch.randn(p + n, CTOR['dim'], generator=g), torch.randn(p + n, 3, generator=g) * 3) for p, n in zip(prompts, gens)]
    return prompts, gens, data


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def packed(model, prompts, gens, data, S):
    """(a): returns (per-request outputs, step seconds)."""
    dec = model.packed_decoder()
    waiting, live, outs, steps = list(range(len(prompts))), {}, [[] for _ in prompts], []
    while waiting or live:
        while waiting and len(live) < S:
            r = waiting.pop(0)
            live[r] = [dec.open()[0], 0]
        reqs = list(live)
        ms = [prompts[r] if live[r][1] == 0 else 1 for r in reqs]
        f = torch.cat([data[r][0][live[r][1]:live[r][1] + m] for r, m in zip(reqs, ms)])
        c = torch.cat([data[r][1][live[r][1]:live[r][1] + m] for r, m in zip(reqs, ms)])
        out, dt = timed(lambda: dec.extend([live[r][0] for r in reqs], ms, f, c))
        steps.append(dt)
        at = 0
        for r, m in zip(reqs, ms):
            outs[r].append(out[at:at + m])
            at += m
            live[r][1] += m
            if live[r][1] == prompts[r] + gens[r]:
                dec.close(live.pop(r)[0])
    return [torch.cat(o) for o in outs], steps


def one_by_one(model, prompts, gens, data):
    """(b)"""
    outs, steps = [], []
    for (f, c), p, n in zip(data, prompts, gens):
        dec = model.causal_decoder(batch_size=1)
        o, dt = timed(lambda: dec.extend(f[None, :p], c[None, :p]))
        rows = [o[0]]
        steps.append(dt)
        for i in range(p, p + n):
            o, dt = timed(lambda: dec.extend(f[None, i:i + 1], c[None, i:i + 1]))
            rows.append(o[0])
            steps.append(dt)
        outs.append(torch.cat(rows))
    return outs, steps


def lockstep(model, prompts, gens, data, S):
    """(c): the steps of static batches of S requests, prompts left-padded to the batch's longest with masked nodes and every
    cloud stepping until the batch's longest request finishes (finished ones on masked nodes)."""
    steps, dev = [], data[0][0].device
    for b0 in range(0, len(prompts), S):
        batch = range(b0, min(b0 + S, len(prompts)))
        P, G = max(prompts[r] for r in batch), max(gens[r] for r in batch)
        feats = torch.zeros(len(batch), P + G, CTOR['dim'], device=dev)
        coors = torch.zeros(len(batch), P + G, 3, device=dev)
        mask = torch.zeros(len(batch), P + G, dtype=torch.bool, device=dev)
        for i, r in enumerate(batch):
            n, pad = prompts[r] + gens[r], P - prompts[r]
            feats[i, pad:pad + n], coors[i, pad:pad + n], mask[i, pad:pad + n] = data[r][0], data[r][1], True
            coors[i, :pad] = data[r][1][:1]
            coors[i, pad + n:] = data[r][1][-1:]
        dec = model.causal_decoder(batch_size=len(batch))
        _, dt = timed(lambda: dec.extend(feats[:, :P], coors[:, :P], mask[:, :P]))
        steps.append(dt)
        for i in range(P, P + G):
            _, dt = timed(lambda: dec.extend(feats[:, i:i + 1], coors[:, i:i + 1], mask[:, i:i + 1]))
            steps.append(dt)
    return steps


def stats(name, steps, wall, generated):
    s = sorted(steps)
    res = dict(wall_s=wall, generated_nodes_per_s=generated / wall, steps=len(s), step_ms_median=1e3 * s[len(s) // 2],
               step_ms_p90=1e3 * s[min(len(s) - 1, int(0.9 * len(s)))], max_memory_allocated_gb=torch.cuda.max_memory_allocated() / 1e9)
    print(f'{name}: {wall:.2f} s, {res["generated_nodes_per_s"]:.1f} generated nodes/s, {len(s)} steps, step median '
          f'{res["step_ms_median"]:.1f} ms, p90 {res["step_ms_p90"]:.1f} ms, peak memory {res["max_memory_allocated_gb"]:.2f} GB', flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--requests', type=int, default=32)
    ap.add_argument('--reps', type=int, default=2, help='timed runs of each schedule, after one warm-up run')
    ap.add_argument('--slots', type=int, nargs='+', default=[4, 16])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_decode_packed.py needs a CUDA device')
    from se3_transformer_pytorch_b200 import SE3Transformer
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    gpu = card()
    print('card, power limit:', gpu, flush=True)
    with torch.device(dev):
        model = SE3Transformer(**CTOR)
    model.eval()
    fill_device(model)
    prompts, gens, data = trace(args.requests)
    data = [(f.to(dev), c.to(dev)) for f, c in data]
    dmax = max(float(torch.cdist(c, c).max()) for _, c in data)
    model.pack_weights(free_master=True, max_distance=1.1 * dmax)
    generated = sum(gens)
    res = dict(card=gpu, ctor=CTOR, requests=args.requests, prompt_range=[min(prompts), max(prompts)],
               generated_range=[min(gens), max(gens)], generated_nodes=generated, runs={})
    print(f'trace: {args.requests} requests, prompts {min(prompts)} .. {max(prompts)}, {generated} generated nodes', flush=True)

    schedules = [(f'a_packed_S{S}', lambda S=S: packed(model, prompts, gens, data, S)) for S in args.slots]
    schedules.append(('b_batch1', lambda: one_by_one(model, prompts, gens, data)))
    schedules += [(f'c_lockstep_S{S}', lambda S=S: (None, lockstep(model, prompts, gens, data, S))) for S in args.slots]
    outputs = {}
    for rep in range(args.reps + 1):                 # rep 0 warms every step shape of every schedule
        for name, run in schedules:
            torch.cuda.reset_peak_memory_stats()
            (outs, steps), wall = timed(run)
            if rep == 0:
                outputs[name] = outs
                continue
            res['runs'].setdefault(name, []).append(stats(f'{name} (run {rep})', steps, wall, generated))
    ref = outputs['b_batch1']
    for S in args.slots:
        got = outputs[f'a_packed_S{S}']
        res[f'a_S{S}_equal_b'] = all(torch.equal(x, y) for x, y in zip(got, ref))
        print(f'(a) S = {S}: every request torch.equal to (b): {res[f"a_S{S}_equal_b"]}', flush=True)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
