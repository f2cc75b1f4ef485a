"""The paged cache of the packed causal decoder (packed_decoder(page_size=16)) against the unpaged one, with bench_decode.py's
model (the README's autoregressive model: dim 512, 8 x 64 heads, depth 6, 4 degrees, valid_radius 10, causal, k = 16), weights
and production path.

    python bench_decode_paged.py [--page-size 16] [--beams 8] [--reps 1] [--schedules a b c]

Schedules, each run once with the profiler's CUDA events on (which times the neighbour search of every step) and then --reps
times timed, the paged and the unpaged decoder alternating:
  (a) mixed trace: 15 requests of bench_decode_packed.py's trace (prompts 256 .. 960, 16 .. 64 generated nodes) beside one
      request with a 4096-node prompt and 64 generated nodes, all 16 in flight, each closing when done;
  (b) beam search: a 4096-node prompt, forked into --beams beams, 64 single-node steps in which every beam extends.  Halfway the
      last half of the beams close and as many new beams fork from the survivors, rewound by 3 nodes (into a page the survivor
      still holds), so that close, truncate and copy-on-write all occur;
  (c) (b) with 32 beams, paged only: the unpaged cache would need 64 rows of 8192 nodes (its growth rule), printed instead.
Every step ends in a device synchronise.  Reports wall time, generated nodes/s, step median and p90, peak
torch.cuda.max_memory_allocated above the resident weights and inputs, pages in use, and the median neighbour-search time per
step; checks that every request's rows are torch.equal between the two decoders; prints a JSON summary with the card and its
power limit."""
import argparse
import json
import sys
import time

import torch

from bench_decode import CTOR, card, fill_device
from bench_decode_packed import trace

PROMPT, GEN = 4096, 64


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def mixed(dec, prompts, gens, data):
    """(a): (per-request outputs, step seconds, pages in use after each step)."""
    ids = dec.open(len(prompts))
    done, outs, steps, pages = [0] * len(prompts), [[] for _ in prompts], [], []
    while any(c is not None for c in ids):
        live = [r for r, c in enumerate(ids) if c is not None]
        ms = [prompts[r] if done[r] == 0 else 1 for r in live]
        f = torch.cat([data[r][0][done[r]:done[r] + m] for r, m in zip(live, ms)])
        c = torch.cat([data[r][1][done[r]:done[r] + m] for r, m in zip(live, ms)])
        out, dt = timed(lambda: dec.extend([ids[r] for r in live], ms, f, c))
        steps.append(dt)
        pages.append(dec.pages_in_use() if hasattr(dec, 'pages_in_use') else None)
        at = 0
        for r, m in zip(live, ms):
            outs[r].append(out[at:at + m])
            at, done[r] = at + m, done[r] + m
            if done[r] == prompts[r] + gens[r]:
                dec.close(ids[r])
                ids[r] = None
    return [torch.cat(o) for o in outs], steps, pages


def beams(dec, prompt, W, steps_n, seed=1):
    """(b) / (c): (every beam's outputs, keyed by beam number, step seconds, pages in use after each step)."""
    g = torch.Generator(device=prompt[0].device).manual_seed(seed)
    root, = dec.open()
    _, dt = timed(lambda: dec.extend([root], [PROMPT], *prompt))
    steps, pages, outs = [dt], [], {}
    live = {b: dec.fork(root) for b in range(W)}
    dec.close(root)
    nxt = W
    for s in range(steps_n):
        if s == steps_n // 2:
            for b in list(live)[W // 2:]:
                dec.close(live.pop(b))
            for b in list(live)[:W - len(live)]:
                live[nxt] = dec.fork(live[b])
                dec.truncate(live[nxt], dec.length(live[nxt]) - 3)
                outs[nxt] = list(outs[b][:-3])
                nxt += 1
        bs = list(live)
        f = torch.randn(len(bs), CTOR['dim'], generator=g, device=g.device)
        c = torch.randn(len(bs), 3, generator=g, device=g.device) * 3
        out, dt = timed(lambda: dec.extend([live[b] for b in bs], [1] * len(bs), f, c))
        steps.append(dt)
        pages.append(dec.pages_in_use() if hasattr(dec, 'pages_in_use') else None)
        for i, b in enumerate(bs):
            outs.setdefault(b, []).append(out[i:i + 1])
    return {b: torch.cat(o) for b, o in outs.items()}, steps, pages


def unpaged_bytes(rows, nodes, per_node):
    """The unpaged cache after its growth rule (each axis doubled when full, from 16 nodes) for `rows` clouds of at most `nodes`."""
    S, cap = 1, 16
    while S < rows:
        S *= 2
    while cap < nodes:
        cap *= 2
    return S * cap * per_node


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--page-size', type=int, default=16)
    ap.add_argument('--beams', type=int, default=8)
    ap.add_argument('--reps', type=int, default=1, help='timed runs of each schedule, after one profiled run')
    ap.add_argument('--schedules', nargs='+', default=['a', 'b', 'c'])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_decode_paged.py needs a CUDA device')
    from se3_transformer_pytorch_b200 import SE3Transformer, ops
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    gpu = card()
    print('card, power limit:', gpu, flush=True)
    with torch.device(dev):
        model = SE3Transformer(**CTOR)
    model.eval()
    fill_device(model)
    prompts, gens, data = trace(15)
    g = torch.Generator().manual_seed(7)
    data.append((torch.randn(PROMPT + GEN, CTOR['dim'], generator=g), torch.randn(PROMPT + GEN, 3, generator=g) * 3))
    prompts, gens = prompts + [PROMPT], gens + [GEN]
    data = [(f.to(dev), c.to(dev)) for f, c in data]
    prompt = data[-1][0][:PROMPT], data[-1][1][:PROMPT]
    dmax = max(float(torch.cdist(c, c).max()) for _, c in data)
    model.pack_weights(free_master=True, max_distance=1.5 * dmax)      # beams draw new nodes beyond the prompt's
    torch.cuda.synchronize()
    resident = torch.cuda.memory_allocated()
    P = args.page_size
    res = dict(card=gpu, ctor=CTOR, page_size=P, runs={})
    schedules = []
    if 'a' in args.schedules:
        schedules += [('a', kind, lambda dec: mixed(dec, prompts, gens, data), sum(gens)) for kind in ('unpaged', 'paged')]
    if 'b' in args.schedules:
        schedules += [('b', kind, lambda dec: beams(dec, prompt, args.beams, GEN), args.beams * GEN) for kind in ('unpaged', 'paged')]
    if 'c' in args.schedules:
        schedules.append(('c', 'paged', lambda dec: beams(dec, prompt, 32, GEN), 32 * GEN))
    outputs = {}
    for rep in range(args.reps + 1):                 # rep 0 warms every step shape and times the neighbour search
        for sched, kind, run, generated in schedules:
            dec = None                               # the previous decoder's cache is freed before this one allocates
            dec = model.packed_decoder(page_size=P if kind == 'paged' else None)
            torch.cuda.reset_peak_memory_stats()
            ops.PROFILE = [] if rep == 0 else None
            try:
                (outs, steps, pages), wall = timed(lambda: run(dec))
                prof = ops.PROFILE
            finally:
                ops.PROFILE = None
            key = f'{sched}_{kind}'
            if rep == 0:
                outputs[key] = outs
                search = sorted(s.elapsed_time(e) for name, s, e, *_ in prof if name.startswith('knn_rows'))
                res.setdefault('search_ms_median', {})[key] = search[len(search) // 2]
                print(f'{key}: neighbour search median {search[len(search) // 2]:.3f} ms over {len(search)} steps', flush=True)
                continue
            s = sorted(steps)
            r = dict(wall_s=wall, generated_nodes_per_s=generated / wall, steps=len(s), step_ms_median=1e3 * s[len(s) // 2],
                     step_ms_p90=1e3 * s[min(len(s) - 1, int(0.9 * len(s)))],
                     peak_gb_above_resident=(torch.cuda.max_memory_allocated() - resident) / 1e9)
            if kind == 'paged':
                r.update(pages_in_use_end=pages[-1], pages_in_use_max=max(pages), pages_reserved=dec.pages_reserved(),
                         cache_gb_reserved=dec.pages_reserved() * P * dec.cache_bytes_per_node() / 1e9)
            res['runs'].setdefault(key, []).append(r)
            print(f'{key} (run {rep}): {json.dumps(r)}', flush=True)
            if sched == 'c':
                per_node = dec.cache_bytes_per_node()
                res['c_unpaged_cache_gb_from_growth_rule'] = unpaged_bytes(33, PROMPT + GEN, per_node) / 1e9
    for sched in ('a', 'b'):
        if f'{sched}_paged' in outputs:
            got, want = outputs[f'{sched}_paged'], outputs[f'{sched}_unpaged']
            keys = range(len(got)) if isinstance(got, list) else sorted(got)
            res[f'{sched}_paged_equal_unpaged'] = sorted(keys) == sorted(range(len(want)) if isinstance(want, list) else want) and \
                all(torch.equal(got[k], want[k]) for k in keys)
            print(f'({sched}) every request torch.equal paged vs unpaged: {res[f"{sched}_paged_equal_unpaged"]}', flush=True)
    if 'c_unpaged_cache_gb_from_growth_rule' in res:
        print(f'(c) the unpaged cache would need {res["c_unpaged_cache_gb_from_growth_rule"]:.1f} GB (64 rows x 8192 nodes)', flush=True)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
