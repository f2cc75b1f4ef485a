"""Generation with the README's autoregressive model (dim 512, 8 x 64 heads, depth 6, 4 degrees, valid_radius 10, causal, k = 16):
the cost of one CausalDecoder step at a 960 .. 1023-node prefix, at batch 1 and at batch 4 in lockstep, against one full forward
of 1024 nodes (what a step costs without the cache), and the step's production GEMMs split-K against unsplit.

    python bench_decode.py [--steps 64] [--warmup 8] [--prefill 960]

Prints one line per measurement and a JSON summary.  Weights follow the magnitudes of tests/golden/detfill.py, drawn on the device
from a generator seeded by the crc32 of each state_dict key (the numpy fill would take minutes at this width)."""
import argparse
import json
import subprocess
import sys
import time
import zlib

import torch

CTOR = dict(dim=512, heads=8, dim_head=64, depth=6, num_degrees=4, num_neighbors=16, valid_radius=10, causal=True)


def fill_device(model, seed=0):
    """detfill's magnitudes (det_tensor) with device-generated normals."""
    with torch.no_grad():
        for key, v in model.state_dict().items():
            if not torch.is_floating_point(v) or key.endswith('inv_freq'):
                continue
            g = torch.Generator(device=v.device).manual_seed(zlib.crc32(key.encode()) * 7919 + seed)
            z = torch.randn(v.shape, generator=g, device=v.device, dtype=v.dtype)
            parts, leaf = key.split('.'), key.split('.')[-1]
            if 'rp' in parts and parts[parts.index('rp') + 2] in ('1', '4'):
                z = 1.0 + 0.1 * z if leaf == 'weight' else 0.1 * z
            elif 'rp' in parts:
                z = 0.1 * z if leaf == 'bias' else z / v.shape[1] ** 0.5
            elif leaf == 'scale':
                z = 1.0 + 0.1 * z
            elif 'weights' in parts:
                z = z / v.shape[0] ** 0.5
            v.copy_(z)


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                          str(torch.cuda.current_device())], capture_output=True, text=True)
    return out.stdout.strip() or 'unknown'


def decode(model, feats, coors, prefill, steps):
    """(per-step seconds, outputs of every call concatenated): prefill nodes, then `steps` single-node steps."""
    dec = model.causal_decoder(batch_size=feats.shape[0])
    outs = [dec.extend(feats[:, :prefill], coors[:, :prefill])]
    times = []
    for i in range(prefill, prefill + steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        outs.append(dec.extend(feats[:, i:i + 1], coors[:, i:i + 1]))
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    if torch.is_tensor(outs[0]):
        return times, torch.cat(outs, dim=1), dec
    return times, {d: torch.cat([o[d] for o in outs], dim=1) for d in outs[0]}, dec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=64)
    ap.add_argument('--warmup', type=int, default=8)
    ap.add_argument('--prefill', type=int, default=960)
    ap.add_argument('--reps', type=int, default=20, help='alternating repetitions of the GEMM comparison')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_decode.py needs a CUDA device')
    from se3_transformer_pytorch_b200 import SE3Transformer, ops
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    gpu = card()
    print('card, power limit:', gpu, flush=True)
    with torch.device(dev):
        model = SE3Transformer(**CTOR)
    model.eval()
    fill_device(model)
    n = args.prefill + args.steps
    g = torch.Generator().manual_seed(7)
    feats = torch.randn(4, n, CTOR['dim'], generator=g).to(dev)
    coors = (torch.randn(4, n, 3, generator=g) * 3).to(dev)
    model.pack_weights(free_master=True, max_distance=1.1 * float(torch.cdist(coors, coors).max()))
    torch.cuda.synchronize()
    res = dict(card=gpu, ctor=CTOR, prefill=args.prefill, steps=args.steps)

    for b in (1, 4):
        decode(model, feats[:b], coors[:b], args.prefill, args.warmup)              # warm-up steps
        times, out, dec = decode(model, feats[:b], coors[:b], args.prefill, args.steps)
        ms = 1e3 * sum(times) / len(times)
        res[f'step_ms_b{b}'] = ms
        print(f'batch {b}: {args.steps} steps at prefix {args.prefill} .. {n - 1}: {ms:.3f} ms/step '
              f'(first {1e3 * times[0]:.3f}, last {1e3 * times[-1]:.3f}); cache {dec.cache_bytes_per_node()} B/node/cloud', flush=True)
        if b == 1:
            decoded = out

    # the full forward a step would cost without the cache, and what it computes for the same rows
    for _ in range(2):
        full = model(feats[:1], coors[:1])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(3):
        full = model(feats[:1], coors[:1])
    torch.cuda.synchronize()
    res['full_forward_ms_b1'] = 1e3 * (time.perf_counter() - t0) / 3
    res['decoded_equal_forward'] = torch.equal(decoded, full)
    print(f'full forward of {n} nodes (batch 1): {res["full_forward_ms_b1"]:.1f} ms; decoded rows torch.equal forward: '
          f'{res["decoded_equal_forward"]}', flush=True)

    # one step's production GEMMs (and LinearSE3 images) as launched, then replayed split and unsplit, alternating
    dec = model.causal_decoder(batch_size=1)
    dec.extend(feats[:1, :n - 1], coors[:1, :n - 1])
    calls, lin_bytes = [], [0]
    zgemm, linear_tc = ops.zgemm, ops.linear_tc

    def rec_zgemm(*a, **kw):
        calls.append((a, kw))
        return zgemm(*a, **kw)

    def rec_linear(x, img, *a, **kw):
        lin_bytes[0] += img.numel()
        return linear_tc(x, img, *a, **kw)
    ops.zgemm, ops.linear_tc = rec_zgemm, rec_linear
    ops.PROFILE = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    try:
        dec.extend(feats[:1, n - 1:n], coors[:1, n - 1:n])
        torch.cuda.synchronize()
    finally:
        ops.zgemm, ops.linear_tc = zgemm, linear_tc
        prof, ops.PROFILE = ops.PROFILE, None
    wall = 1e3 * (time.perf_counter() - t0)
    kinds = {}
    for name, s, e, *_ in prof:
        kinds[name] = kinds.get(name, 0.0) + s.elapsed_time(e)
    res['profiled_step_ms'] = wall
    res['kernel_ms_by_kind'] = kinds
    print(f'profiled step (batch 1, prefix {n - 1}): {wall:.3f} ms wall, {len(prof)} launches; kernel ms by kind: '
          + ', '.join(f'{k} {v:.3f}' for k, v in sorted(kinds.items(), key=lambda kv: -kv[1])), flush=True)

    def run_all(k):
        for a, kw in calls:
            zgemm(*a, **dict(kw, k_split=k))
    chosen = []
    for a, kw in calls:
        E, Co, mode = a[3], a[4], a[5]
        arr = (ops.ZSeg * len(a[0]))(*[ops.ZSeg(U.data_ptr(), X.data_ptr(), Ci, nc, cp, cm) for U, X, Ci, nc, cp, cm in a[0]])
        units = ops.lib().se3_zgemm_split_units(arr, len(a[0]), Co, mode, kw.get('flush_stages', 0))
        chosen.append(ops.zgemm_k_split((E + 127) // 128 * (Co // 128), units, ops.sm_count(dev)))
    t = {1: [], 'auto': []}
    for _ in range(2):
        run_all(1)
        run_all(None)
    for _ in range(args.reps):
        for k in (1, None):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            run_all(k)
            e.record()
            e.synchronize()
            t[1 if k == 1 else 'auto'].append(s.elapsed_time(e))
    med = lambda v: sorted(v)[len(v) // 2]
    img_bytes = sum(a[1].numel() for a, _ in calls)
    res.update(step_gemms=len(calls), k_split_chosen=sorted(set(chosen)), gemm_ms_unsplit=med(t[1]), gemm_ms_split=med(t['auto']),
               gemm_ms_spread_unsplit=[min(t[1]), max(t[1])], gemm_ms_spread_split=[min(t['auto']), max(t['auto'])],
               zgemm_image_bytes=img_bytes, linear_image_bytes=lin_bytes[0])
    print(f'{len(calls)} production GEMMs of one step (k_split chosen {sorted(set(chosen))}): unsplit {res["gemm_ms_unsplit"]:.3f} ms, '
          f'split {res["gemm_ms_split"]:.3f} ms (medians of {args.reps}, alternating)', flush=True)
    total = img_bytes + lin_bytes[0]
    for b in (1, 4):
        rate = total / (res[f'step_ms_b{b}'] * 1e-3) / 1e12
        print(f'batch {b}: weight-image bytes per step {total / 1e9:.2f} GB / step time = effective rate {rate:.3f} TB/s')
        res[f'effective_image_tb_s_b{b}'] = rate
    print(json.dumps(res))


if __name__ == '__main__':
    main()
