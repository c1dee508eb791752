"""The fp8 decoder mode against fp16 on the headline workload: B = 64 encode + 50-step decode, FULL dims, synthetic weights.

1. speed      fp16 and fp8 alternated 3x on the same seeded batch, CUDA events around encode + decode (graphs on, as
              bench.py runs them); images/s per run.  The SM clock is read after every run; its median is reported.
2. accuracy   the 50-step latents of fp8 and of fp16 against bf16x3 on the same seeded inputs (max-abs and RMS), and the
              Engine auto-probe's figure -- max-abs velocity deviation against bf16x3 at the first and the last step on its
              seeded probe image.
The GPU name and power limit are read in the same run.  Prints a table and one JSON line; --out DIR also writes it there.

    python profiles/fp8_bench.py [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from selftoktokenizer_b200 import config as C, synth  # noqa: E402
from selftoktokenizer_b200.capi import Engine  # noqa: E402

B, STEPS, ROUNDS = 64, 50, 3


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30, check=True)
    return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().split(",")]))


def sm_clock_mhz():
    return float(gpu_info()["clocks.sm"].split()[0])


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def probe_dev(eng, ref, d):
    """the Engine auto-probe's figure: max-abs velocity deviation against `ref` at the first and last step"""
    from selftoktokenizer_b200 import synth as sy
    x = sy.synth_tensor("auto.probe.x", (1, d.in_channels, d.latent, d.latent), "emb", 1.0)
    tok = (torch.arange(d.K, dtype=torch.int64) * 2654435761 % d.codebook_size).reshape(1, d.K)
    return {st: float((eng.dit_velocity(tok, x, st) - ref.dit_velocity(tok, x, st)).abs().max()) for st in (0, STEPS - 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_bench.py needs a CUDA device")
    d, dev = C.FULL, torch.device("cuda:0")
    sd = synth.synth_state_dict(d, device=dev)
    g = torch.Generator().manual_seed(0)
    x0 = torch.randn(B, d.in_channels, d.latent, d.latent, generator=g).to(dev)
    noise = torch.randn(B, d.in_channels, d.latent, d.latent, generator=g).to(dev)
    engines = {p: Engine(d, sd, device=dev, precision=p, steps=STEPS) for p in ("fp16", "fp8")}
    tok = engines["fp16"].encode(x0)
    lat = {}
    for p, e in engines.items():                               # warm-up: graphs captured, workspaces placed
        e.encode(x0)
        lat[p] = e.decode(tok, noise).cpu()
    torch.cuda.synchronize()
    runs = {p: [] for p in engines}
    clocks = []
    for _ in range(ROUNDS):
        for p, e in engines.items():
            ms = timed(lambda: (e.encode(x0), e.decode(tok, noise)))
            runs[p].append(B / (ms / 1e3))
            clocks.append(sm_clock_mhz())
    ref = Engine(d, sd, device=dev, precision="bf16x3", steps=STEPS)
    lat["bf16x3"] = ref.decode(tok, noise).cpu()
    acc = {}
    for p, e in engines.items():
        diff = (lat[p] - lat["bf16x3"]).double()
        acc[p] = {"latent_max_abs": float(diff.abs().max()), "latent_rms": float(diff.pow(2).mean().sqrt()),
                  "velocity_max_abs": probe_dev(e, ref, d)}
    for e in (*engines.values(), ref):
        e.close()
    spread = {p: max(v) - min(v) for p, v in runs.items()}
    mean = {p: statistics.mean(v) for p, v in runs.items()}
    out = {"gpu": gpu_info(), "batch": B, "steps": STEPS, "images_per_s": runs, "mean": mean, "spread": spread,
           "speedup": mean["fp8"] / mean["fp16"], "median_sm_clock_mhz": statistics.median(clocks),
           "accuracy_vs_bf16x3": acc}
    print(f"{out['gpu']['name']}, power limit {out['gpu']['power.limit']}, median SM clock {out['median_sm_clock_mhz']:.0f} MHz")
    for p in runs:
        print(f"{p:>6}: images/s {' / '.join(f'{v:.3f}' for v in runs[p])} (mean {mean[p]:.3f}, spread {spread[p]:.3f}); "
              f"latents vs bf16x3 max-abs {acc[p]['latent_max_abs']:.3e} RMS {acc[p]['latent_rms']:.3e}; "
              f"velocity vs bf16x3 {acc[p]['velocity_max_abs']}")
    print(f"fp8 / fp16: {out['speedup']:.3f}x")
    print(json.dumps(out))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(out, open(os.path.join(a.out, "fp8_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
