"""One engine serving several image sizes against a dedicated engine per size: FULL dims, fp16, synthetic weights.

1. throughput  images/s of encode + 50-step decode at 128^2, 256^2, 384^2, 512^2 and 512 x 256 pixels: the one engine (built at
               256^2, `latent_hw=` per call) and a dedicated engine per square size, alternated, ROUNDS times.  B per size keeps
               the image tokens per batch at the headline's (B = 64 at 256^2), capped at 256.  CUDA events around each call, graphs
               on as bench.py runs them; the SM clock is read after every run and its median reported.
2. first call  wall time of the one engine's first encode + decode at each new size (positional crops, workspace growth, graph
               capture) against its steady-state time.
3. memory      selftok_device_bytes of the one engine after serving every size against the sum over the dedicated engines.
The GPU name and power limit are read in the same run.  Prints a table and one JSON line; --out DIR also writes it there.

    python profiles/size_bench.py [--rounds 3] [--out DIR]
"""
import argparse
import dataclasses
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fp8_bench import gpu_info, sm_clock_mhz, timed  # noqa: E402
from selftoktokenizer_b200 import config as C, synth  # noqa: E402
from selftoktokenizer_b200.capi import Engine  # noqa: E402

PIXELS = [(128, 128), (256, 256), (384, 384), (512, 512), (512, 256)]
STEPS = 50


def batch_for(hw, d):
    return max(1, min(256, 64 * d.latent * d.latent // ((hw[0] // 8) * (hw[1] // 8))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("size_bench.py needs a CUDA device")
    d, dev = C.FULL, torch.device("cuda:0")
    sd = synth.synth_state_dict(d, device=dev)
    g = torch.Generator().manual_seed(0)
    work = {}
    for px in PIXELS:
        hw = (px[0] // 8, px[1] // 8)
        B = batch_for(px, d)
        work[px] = (hw, B, torch.randn(B, d.in_channels, *hw, generator=g).to(dev), torch.randn(B, d.in_channels, *hw, generator=g).to(dev))
    one = Engine(d, sd, device=dev, precision="fp16", steps=STEPS)

    def run(eng, px, own):
        hw, B, x0, noise = work[px]
        lh = None if own else hw
        tok = eng.encode(x0, latent_hw=lh)
        eng.decode(tok, noise, latent_hw=lh)

    first = {}
    for px in PIXELS:                                   # first call at each size: crops, workspace growth, graph capture
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run(one, px, False)
        torch.cuda.synchronize()
        first[px] = time.perf_counter() - t0
    one_bytes = one.device_bytes
    own = {}
    own_bytes = 0
    for px in PIXELS:
        if px[0] == px[1]:
            own[px] = Engine(dataclasses.replace(d, latent=px[0] // 8), sd, device=dev, precision="fp16", steps=STEPS)
            run(own[px], px, True)                      # warm-up
            own_bytes += own[px].device_bytes
    runs = {f"{px[0]}x{px[1]}": {"one": [], "dedicated": []} for px in PIXELS}
    clocks = []
    steady = {px: [] for px in PIXELS}
    for _ in range(a.rounds):
        for px in PIXELS:
            B = work[px][1]
            ms = timed(lambda: run(one, px, False))
            steady[px].append(ms / 1e3)
            runs[f"{px[0]}x{px[1]}"]["one"].append(B / (ms / 1e3))
            clocks.append(sm_clock_mhz())
            if px in own:
                ms = timed(lambda: run(own[px], px, True))
                runs[f"{px[0]}x{px[1]}"]["dedicated"].append(B / (ms / 1e3))
                clocks.append(sm_clock_mhz())
    for e in (one, *own.values()):
        e.close()
    out = {"gpu": gpu_info(), "steps": STEPS, "median_sm_clock_mhz": statistics.median(clocks),
           "batch": {f"{px[0]}x{px[1]}": work[px][1] for px in PIXELS}, "images_per_s": runs,
           "first_call_s": {f"{px[0]}x{px[1]}": first[px] for px in PIXELS},
           "steady_call_s": {f"{px[0]}x{px[1]}": statistics.median(steady[px]) for px in PIXELS},
           "device_bytes": {"one_engine": one_bytes, "dedicated_sum": own_bytes}}
    print(f"{out['gpu']['name']}, power limit {out['gpu']['power.limit']}, median SM clock {out['median_sm_clock_mhz']:.0f} MHz")
    for px in PIXELS:
        k = f"{px[0]}x{px[1]}"
        r = runs[k]
        ded = " / ".join(f"{v:.3f}" for v in r["dedicated"]) or "-"
        print(f"{k:>8} B={work[px][1]:>3}: images/s one engine {' / '.join(f'{v:.3f}' for v in r['one'])}; dedicated {ded}; "
              f"first call {first[px]:.2f} s vs steady {out['steady_call_s'][k]:.2f} s")
    print(f"device bytes: one engine {one_bytes / 2**30:.2f} GiB, dedicated engines (4 square sizes) {own_bytes / 2**30:.2f} GiB")
    print(json.dumps(out))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(out, open(os.path.join(a.out, "size_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
