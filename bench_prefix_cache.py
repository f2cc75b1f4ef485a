"""The prefix cache of the paged decoder (packed_decoder(page_size=16, max_nodes=..., prefix_cache=True), DESIGN.md 10.4) against
the same decoder without it, with bench_decode.py's model (the README's autoregressive model: dim 512, 8 x 64 heads, depth 6,
4 degrees, valid_radius 10, causal, k = 16), weights and production path.

    python bench_prefix_cache.py [--requests 16] [--prompt 4096] [--tail 32] [--gen 32] [--page-size 16] [--reps 1]

Schedule: --requests requests, each a shared --prompt-node prompt followed by its own --tail-node tail, arriving one per step
(request r joins at step r with its whole prompt and tail in one call), every request already in flight generating one node per
step, --gen generated nodes each, then closing.  The pool holds max_nodes = requests x (prompt + tail + gen) nodes, so the run
without the cache fits.  One warm-up run of each, then --reps timed runs, the cache on and off alternating in one process.
Every step ends in a device synchronise.  Reports each request's time to first rows (the step that carries its prompt), wall
time, generated nodes/s, the median of the prompt steps and of the decode steps, peak torch.cuda.max_memory_allocated above
the resident weights and inputs, and pages reserved / in use (max) / cached (end); checks that every request's rows are
torch.equal between the two decoders; prints a JSON summary with the card and its power limit."""
import argparse
import json
import sys
import time

import torch

from bench_decode import CTOR, card, fill_device


def run(dec, data, prompt_len, gen):
    """(every request's rows, time to first rows and nodes from the cache per request, prompt-step and decode-step seconds, max
    pages in use)."""
    R = len(data)
    ids, done, outs, first, cached = [None] * R, [0] * R, [[] for _ in range(R)], [None] * R, [0] * R
    prompt_steps, decode_steps, in_use = [], [], 0
    step = 0
    while step < R or any(c is not None for c in ids):
        if step < R:
            ids[step] = dec.open()[0]
        live = [r for r in range(R) if ids[r] is not None]
        ms = [prompt_len if done[r] == 0 else 1 for r in live]
        f = torch.cat([data[r][0][done[r]:done[r] + m] for r, m in zip(live, ms)])
        c = torch.cat([data[r][1][done[r]:done[r] + m] for r, m in zip(live, ms)])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = dec.extend([ids[r] for r in live], ms, f, c)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        (prompt_steps if step < R else decode_steps).append(dt)
        in_use = max(in_use, dec.pages_in_use())
        at = 0
        for r, m in zip(live, ms):
            outs[r].append(out[at:at + m])
            if done[r] == 0:
                first[r], cached[r] = dt, dec.prefix_nodes(ids[r])
            at, done[r] = at + m, done[r] + m
            if done[r] == prompt_len + gen:
                dec.close(ids[r])
                ids[r] = None
        step += 1
    return [torch.cat(o) for o in outs], first, cached, prompt_steps, decode_steps, in_use


def median(v):
    s = sorted(v)
    return s[len(s) // 2] if s else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--requests', type=int, default=16)
    ap.add_argument('--prompt', type=int, default=4096, help='nodes of the prompt every request shares')
    ap.add_argument('--tail', type=int, default=32, help='nodes of each request\'s own prompt tail')
    ap.add_argument('--gen', type=int, default=32, help='generated nodes per request')
    ap.add_argument('--page-size', type=int, default=16)
    ap.add_argument('--reps', type=int, default=1, help='timed runs of each decoder, after one warm-up run')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_prefix_cache.py needs a CUDA device')
    from se3_transformer_pytorch_b200 import SE3Transformer
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    gpu = card()
    print('card, power limit:', gpu, flush=True)
    with torch.device(dev):
        model = SE3Transformer(**CTOR)
    model.eval()
    fill_device(model)
    R, n = args.requests, args.prompt + args.tail + args.gen
    g = torch.Generator().manual_seed(11)
    shared = torch.randn(args.prompt, CTOR['dim'], generator=g), torch.randn(args.prompt, 3, generator=g) * 3
    data = []
    for _ in range(R):
        own = torch.randn(n - args.prompt, CTOR['dim'], generator=g), torch.randn(n - args.prompt, 3, generator=g) * 3
        data.append((torch.cat([shared[0], own[0]]).to(dev), torch.cat([shared[1], own[1]]).to(dev)))
    dmax = max(float(torch.cdist(c, c).max()) for _, c in data)
    model.pack_weights(free_master=True, max_distance=1.5 * dmax)
    P, max_nodes = args.page_size, R * n
    prompt_len = args.prompt + args.tail
    torch.cuda.synchronize()
    res = dict(card=gpu, ctor=CTOR, page_size=P, max_nodes=max_nodes, requests=R, prompt=args.prompt, tail=args.tail,
               gen=args.gen, runs={})
    outputs = {}
    for rep in range(args.reps + 1):                 # rep 0 warms every step shape and captures the decode graphs
        for cache in (True, False):
            key = 'cache' if cache else 'no_cache'
            dec = None                               # the previous decoder's pool is freed before this one allocates
            torch.cuda.empty_cache()
            resident = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            dec = model.packed_decoder(page_size=P, max_nodes=max_nodes, prefix_cache=cache)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            outs, first, cached, prompt_steps, decode_steps, in_use = run(dec, data, prompt_len, args.gen)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            if rep == 0:
                outputs[key] = [o.cpu() for o in outs]
            r = dict(wall_s=wall, generated_nodes_per_s=R * args.gen / wall,
                     first_rows_s=[round(v, 4) for v in first], first_rows_s_median=median(first),
                     prompt_step_ms_median=1e3 * median(prompt_steps), decode_step_ms_median=1e3 * median(decode_steps),
                     peak_gb_above_resident=(torch.cuda.max_memory_allocated() - resident) / 1e9,
                     pages_reserved=dec.pages_reserved(), pages_in_use_max=in_use, pages_in_use_end=dec.pages_in_use(),
                     pages_cached_end=dec.pages_cached(), graph_replays=dec.graph_replays, nodes_from_cache=cached)
            res['runs'].setdefault(key, []).append(dict(r, warmup=rep == 0))
            print(f'{key} ({"warm-up" if rep == 0 else f"run {rep}"}): {json.dumps(r)}', flush=True)
            if rep > 0:
                got = [o.cpu() for o in outs]
                same = all(torch.equal(a, b) for a, b in zip(got, outputs[key]))
                res.setdefault('equal_to_warmup', []).append(same)
    equal = all(torch.equal(a, b) for a, b in zip(outputs['cache'], outputs['no_cache']))
    res['every_request_equal'] = equal
    print(f'every request torch.equal with and without the cache: {equal}', flush=True)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
