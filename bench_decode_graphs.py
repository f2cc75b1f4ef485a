"""Paged decoding steps replayed from CUDA graphs against the same steps run eagerly (SE3B200_NO_DECODE_GRAPHS), with
bench_decode.py's model (dim 512, 8 x 64 heads, depth 6, 4 degrees, valid_radius 10, causal, k = 16), weights and production
path, on packed_decoder(page_size=16, max_nodes=...) (DESIGN.md 10.3).

    python bench_decode_graphs.py [--page-size 16] [--reps 3] [--schedules a b8 b32]

Schedules (bench_decode_paged.py's):
  (a)   the decode-only phase of its mixed trace: 16 requests join with their prompts in the first step (eager, not timed), then
        every step carries one node of each live request;
  (b8)  beam search over a 4096-node prompt with 8 beams, 64 single-node steps with a close / fork / truncate halfway;
  (b32) the same with 32 beams.
Each decoder lives across the runs: run 0 warms it (and captures every bucket of the graphed one); runs 1 .. reps are timed,
graphed and eager alternating, every step ending in a device synchronise.  Reports step median and p90 and generated nodes/s
over the decode steps, the capture time of each bucket, the memory each decoder holds with no cloud open (pool, graphs and
their buffers) and the peak above that during a run; then, in a separate run under torch.profiler, device time per step.
Checks that every request's rows are torch.equal across the two paths and prints a JSON summary with the card and its power
limit."""
import argparse
import json
import sys
import time

import torch

from bench_decode import CTOR, card, fill_device
from bench_decode_packed import trace
from bench_decode_paged import GEN, PROMPT, beams, mixed


def close_all(dec):
    for c in dec.open_ids():
        dec.close(c)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--page-size', type=int, default=16)
    ap.add_argument('--reps', type=int, default=3, help='timed runs of each schedule and path, after one warm-up run')
    ap.add_argument('--schedules', nargs='+', default=['a', 'b8', 'b32'])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_decode_graphs.py needs a CUDA device')
    from se3_transformer_pytorch_b200 import SE3Transformer, switches
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
    model.pack_weights(free_master=True, max_distance=1.5 * dmax)
    P = args.page_size
    schedules = {}
    if 'a' in args.schedules:
        schedules['a'] = (lambda dec: mixed(dec, prompts, gens, data), sum(gens), sum(prompts) + sum(gens) + 32 * P)
    for W in (8, 32):
        if f'b{W}' in args.schedules:
            schedules[f'b{W}'] = (lambda dec, W=W: beams(dec, prompt, W, GEN), W * GEN, PROMPT + 2 * W * (GEN + 2 * P))
    torch.cuda.synchronize()
    res = dict(card=gpu, ctor=CTOR, page_size=P, runs={}, capture_s={}, held_gb={}, device_ms_per_step={}, equal={})
    for name, (run, generated, max_nodes) in schedules.items():
        decs, outs = {}, {}
        for kind in ('graphs', 'eager'):          # run 0: warm-up, every bucket captured
            base = torch.cuda.memory_allocated()
            decs[kind] = model.packed_decoder(page_size=P, max_nodes=max_nodes)
            with switches.override(no_decode_graphs=kind == 'eager'):
                outs[kind] = run(decs[kind])[0]
            close_all(decs[kind])
            torch.cuda.synchronize()
            res['held_gb'][f'{name}_{kind}'] = (torch.cuda.memory_allocated() - base) / 1e9
        res['capture_s'][name] = {f'{rows}x{K}': s for (rows, K), s in sorted(decs['graphs'].graph_capture_s.items())}
        got, want = outs['graphs'], outs['eager']
        keys = range(len(got)) if isinstance(got, list) else sorted(got)
        res['equal'][name] = len(got) == len(want) and all(torch.equal(got[k], want[k]) for k in keys)
        print(f'{name}: every request torch.equal graphed vs eager: {res["equal"][name]}; captures (s): {res["capture_s"][name]}',
              flush=True)
        for rep in range(1, args.reps + 1):
            for kind in ('graphs', 'eager'):
                dec = decs[kind]
                replays = dec.graph_replays
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                with switches.override(no_decode_graphs=kind == 'eager'):
                    t0 = time.perf_counter()
                    _, steps, _ = run(dec)
                    torch.cuda.synchronize()
                    wall = time.perf_counter() - t0
                close_all(dec)
                s = sorted(steps[1:])                  # the decode steps: the first one carries the prompts
                r = dict(steps=len(s), step_ms_median=1e3 * s[len(s) // 2], step_ms_p90=1e3 * s[min(len(s) - 1, int(0.9 * len(s)))],
                         generated_nodes_per_s=generated / sum(s), wall_s=wall, replays=dec.graph_replays - replays,
                         peak_gb_above_held=(torch.cuda.max_memory_allocated() - base) / 1e9)
                res['runs'].setdefault(f'{name}_{kind}', []).append(r)
                print(f'{name}_{kind} (run {rep}): {json.dumps(r)}', flush=True)
        for kind in ('graphs', 'eager'):                # device time per step, in a run of its own
            dec = decs[kind]
            with switches.override(no_decode_graphs=kind == 'eager'):
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    _, steps, _ = run(dec)
                    torch.cuda.synchronize()
            close_all(dec)
            total_us = sum(e.self_device_time_total for e in prof.key_averages())
            res['device_ms_per_step'][f'{name}_{kind}'] = total_us / 1e3 / len(steps)
            print(f'{name}_{kind}: device time {total_us / 1e3 / len(steps):.2f} ms per step (prompt step included) over '
                  f'{len(steps)} steps', flush=True)
        del decs, outs
    print(json.dumps(res))


if __name__ == '__main__':
    main()
