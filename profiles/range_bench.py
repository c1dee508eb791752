"""Timing of token-range decodes (selftok_decode_range) at full geometry: B = 64, fp16, CUDA graphs on.

Workloads: selftok_decode against selftok_decode_range with [0, K) (alternated three times: the two must cost the same);
suffix windows (K - n, K), the AR-order reading of n generated tokens, and prefix windows (0, n) for n in {32, 128, 256, 384};
one mixed batch where image b gets the suffix of n = 8 (b + 1) tokens.  Device time by CUDA events around each call, after a
warm-up call of the same window set.  Beside each time: useful FLOPs (each image's own window) and executed FLOPs (the context
stream the call runs: the batch's windows rounded outward to 64 tokens), from schedule.decode_flops_per_image.  The GPU name,
power limit and SM clock are read in the same run.

    python profiles/range_bench.py --out DIR        -> DIR/range_bench.json
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from selftoktokenizer_b200 import config as C, schedule as S, synth  # noqa: E402
from selftoktokenizer_b200.capi import Engine  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().split(",")]))
    except Exception as ex:                                   # the timing itself does not depend on it
        return {"error": str(ex), "name": torch.cuda.get_device_name(0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=2, help="timed calls per window set (the [0, K) guard: one per alternation)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("range_bench needs a CUDA device")
    os.makedirs(a.out, exist_ok=True)
    d, B = C.FULL, a.batch
    eng = Engine(d, synth.synth_state_dict(d, device="cuda:0"), device="cuda:0", precision="fp16")
    tok = ((torch.arange(B * d.K, dtype=torch.int64).reshape(B, d.K) * 2654435761) % d.codebook_size).cuda()
    noise = synth.synth_tensor("range_bench.noise", (B, d.in_channels, d.latent, d.latent), "emb", 1.0).cuda()
    flops = lambda r: S.decode_flops_per_image(d.K, d.stages, d.k_per_stage, 50, d.dit_depth, d.n_img, token_range=r)
    full_eff = S.decode_flops_per_image(d.K, d.stages, d.k_per_stage, 50, d.dit_depth, d.n_img)[0]

    def timed(ranges, reps):
        call = (lambda: eng.decode(tok, noise)) if ranges is None else (lambda: eng.decode(tok, noise, token_range=ranges))
        call()                                                # warm-up: graph capture of this (B, steps, Lo, Hi)
        ms = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return float(np.median(ms)), ms

    def record(name, ranges, reps=a.reps):
        ms, all_ms = timed(ranges, reps)
        rows = np.broadcast_to(np.asarray(ranges if ranges is not None else (0, d.K)), (B, 2))
        useful = sum(flops(tuple(r))[0] for r in rows)
        executed = flops((int(rows[:, 0].min()), int(rows[:, 1].max())))[1] * B
        rec = {"workload": name, "ms_median": ms, "ms": all_ms, "useful_tflop": useful / 1e12, "executed_tflop": executed / 1e12,
               "useful_fraction_of_full": useful / (B * full_eff), "useful_tflops_per_s": useful / 1e12 / (ms / 1e3)}
        print(json.dumps(rec))
        return rec

    out = {"gpu_before": gpu_info(), "geometry": "full (K=512, 32x32 latent), B=%d, fp16, graphs on, 50 steps" % B, "records": []}
    for i in range(3):                                        # regression guard: the plain entry and [0, K), alternated
        out["records"].append(record(f"decode#{i}", None, 1))
        out["records"].append(record(f"decode_range[0,K)#{i}", (0, d.K), 1))
    for n in (32, 128, 256, 384):
        out["records"].append(record(f"suffix n={n}", (d.K - n, d.K)))
    for n in (32, 128, 256, 384):
        out["records"].append(record(f"prefix n={n}", (0, n)))
    mixed = np.array([[d.K - min(d.K, 8 * (b + 1)), d.K] for b in range(B)])
    out["records"].append(record("mixed suffix n=8(b+1)", mixed))
    out["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "range_bench.json"), "w") as f:
        json.dump(out, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
