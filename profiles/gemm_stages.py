"""Per-stage times of the tensor-core GEMM (gemm_tc_kernel) in one full-geometry 50-step decode, graphs off:

    python profiles/gemm_stages.py [precision ...]          # default: fp16 bf16x3

Runs the headline decode (batch 64, FULL dims) once to warm up and once under torch.profiler with CUDA activities, then
attributes every gemm_tc_kernel launch to its stage by its position in the launch sequence.  Per sampler step there are
2 + 4 L launches: x_embedder, then per layer qkv, proj, fc1, fc2 (each one grouped launch of the context and the image
stream), then final_layer.  Algorithmic FLOPs come from the shapes, with the schedule's k_i + 1 visible context rows; the
last layer's context stream is pre_only (qkv only).  Prints one table per precision and one JSON line with the card name,
power limit and SM clock read in the same run.  Needs a GPU; there is no fallback.
"""
import json
import os
import subprocess
import sys
import tempfile

import torch
from torch.profiler import ProfilerActivity, profile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from selftoktokenizer_b200 import capi, config as C, schedule as S, synth  # noqa: E402

B, STEPS = 64, 50
STAGES = ["x_embedder", "qkv", "proj", "fc1", "fc2", "final_layer"]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, plim, sm, smax = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": plim, "sm_clock": sm, "sm_clock_max": smax}


def stage_flops(d):
    """Algorithmic FLOPs of each stage over the whole decode."""
    tb = S.make_tables(d.K, d.stages, d.k_per_stage, STEPS)
    D, N, L = d.dit_hidden, d.n_img, d.dit_depth
    Kp = d.in_channels * d.dit_patch * d.dit_patch
    f = dict.fromkeys(STAGES, 0.0)
    for i in range(STEPS):
        kc = int(tb.k[i]) + 1
        f["x_embedder"] += 2.0 * B * N * Kp * D
        f["final_layer"] += 2.0 * B * N * D * Kp
        for j in range(L):
            rows_ctx = 0 if j == L - 1 else kc
            f["qkv"] += 2.0 * B * (N + kc) * D * 3 * D
            f["proj"] += 2.0 * B * (N + rows_ctx) * D * D
            f["fc1"] += 2.0 * B * (N + rows_ctx) * D * 4 * D
            f["fc2"] += 2.0 * B * (N + rows_ctx) * 4 * D * D
    return f


def gemm_kernel_times(trace_path):
    """Durations (ms) of the gemm_tc_kernel launches in device order."""
    ev = json.load(open(trace_path))["traceEvents"]
    k = [e for e in ev if e.get("cat") == "kernel" and "gemm_tc_kernel" in e.get("name", "")]
    k.sort(key=lambda e: e["ts"])
    return [e["dur"] / 1000.0 for e in k]


def run(prec, tmp):
    d = C.FULL
    dev = torch.device("cuda:0")
    eng = capi.Engine(d, synth.synth_state_dict(d, device=dev), device=dev, precision=prec, steps=STEPS)
    g = torch.Generator().manual_seed(0)
    tok = torch.randint(0, d.codebook_size, (B, d.K), generator=g).to(dev)
    noise = torch.randn(B, d.in_channels, d.latent, d.latent, generator=g).to(dev)
    eng.set_use_graph(False)
    eng.decode(tok, noise)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.decode(tok, noise)
        torch.cuda.synchronize()
    path = os.path.join(tmp, f"gemm_stages_{prec}.pt.trace.json")
    prof.export_chrome_trace(path)
    eng.close()
    times = gemm_kernel_times(path)
    per_step = 2 + 4 * d.dit_depth
    assert len(times) == STEPS * per_step, f"{len(times)} gemm_tc_kernel launches, expected {STEPS} x {per_step}"
    ms = dict.fromkeys(STAGES, 0.0)
    for i, t in enumerate(times):
        p = i % per_step
        ms["x_embedder" if p == 0 else "final_layer" if p == per_step - 1 else STAGES[1 + (p - 1) % 4]] += t
    flops = stage_flops(d)
    total = sum(ms.values())
    rows = {s: {"ms": ms[s], "tflop": flops[s] / 1e12, "tflops": flops[s] / (ms[s] / 1e3) / 1e12, "share": ms[s] / total}
            for s in STAGES}
    rows["all"] = {"ms": total, "tflop": sum(flops.values()) / 1e12,
                   "tflops": sum(flops.values()) / (total / 1e3) / 1e12, "share": 1.0}
    return rows


def main():
    if not torch.cuda.is_available():
        raise SystemExit("gemm_stages.py needs a CUDA device")
    precs = sys.argv[1:] or ["fp16", "bf16x3"]
    out = {"gpu": gpu_info(), "batch": B, "steps": STEPS}
    with tempfile.TemporaryDirectory() as tmp:
        for prec in precs:
            rows = run(prec, tmp)
            out[prec] = rows
            print(f"\n{prec}: gemm_tc_kernel per stage, B = {B}, {STEPS}-step decode, graphs off")
            print(f"{'stage':<12}{'ms':>10}{'TFLOP':>10}{'TFLOP/s':>10}{'share':>8}")
            for s, r in rows.items():
                print(f"{s:<12}{r['ms']:>10.1f}{r['tflop']:>10.1f}{r['tflops']:>10.1f}{r['share']:>8.3f}")
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
