"""Step-level batching (selftok_decode_step / ContinuousDecoder) at full geometry: B = 64, fp16.

1. homogeneous   50 decode_step calls with every image on the same row against selftok_decode (CUDA graph), alternated 3x,
                 CUDA events; the latents must be bitwise equal.  The ratio is the eager per-step overhead.
2. staggered     64 images spread over rows 0..49, each re-admitted at row 0 when done (steady state of a full server); CUDA
                 events around 50 steps after 10 warm-up steps.  images/s = 64 / (50 * step time), its share of (1)'s static
                 images/s, and useful TFLOP/s from schedule.dense_flops_per_image_step over each image's own visible rows.
3. arrivals      256 requests at a constant rate of 0.5x and 0.9x the static throughput, driven in real time (host clock,
                 every completion after a device synchronise): ContinuousDecoder(64) against static batching (fill to 64 or
                 flush after one batch time, then selftok_decode at B = 64).  p50 / p95 latency and completed images/s.
A torch.profiler table of a few staggered steps (device time per kernel) is written beside the JSON.  The GPU name, power
limit and SM clock are read in the same run.

    python profiles/continuous_bench.py --out DIR        -> DIR/continuous_bench.json, DIR/continuous_profile.txt
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from selftoktokenizer_b200 import config as C, schedule as S, synth  # noqa: E402
from selftoktokenizer_b200.capi import Engine  # noqa: E402
from selftoktokenizer_b200.continuous import ContinuousDecoder  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().split(",")]))
    except Exception as ex:                                   # the timing itself does not depend on it
        return {"error": str(ex), "name": torch.cuda.get_device_name(0)}


def events_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--requests", type=int, default=256)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("continuous_bench needs a CUDA device")
    os.makedirs(a.out, exist_ok=True)
    d, B, T = C.FULL, a.batch, 50
    eng = Engine(d, synth.synth_state_dict(d, device="cuda:0"), device="cuda:0", precision="fp16")
    tok = ((torch.arange(B * d.K, dtype=torch.int64).reshape(B, d.K) * 2654435761) % d.codebook_size).cuda()
    noise = synth.synth_tensor("continuous_bench.noise", (B, d.in_channels, d.latent, d.latent), "emb", 1.0).cuda()
    k = eng.tables.k.numpy().astype(np.int64)
    D = 64 * d.dit_depth
    step_flops = [sum(S.dense_flops_per_image_step(D, int(k[s]) + 1, d.n_img, j == d.dit_depth - 1) for j in range(d.dit_depth))
                  for s in range(T)]
    out = {"gpu_before": gpu_info(), "geometry": f"full (K={d.K}, {d.latent}x{d.latent} latent), B={B}, fp16, {T} steps"}

    # ---- 1. homogeneous
    x = noise.clone()

    def steps_loop():
        x.copy_(noise)
        for i in range(T):
            eng.decode_step(tok, x, i, out=x)

    ref = eng.decode(tok, noise)                               # warm-up: graph capture
    steps_loop()
    torch.cuda.synchronize()
    assert torch.equal(x, ref), "homogeneous decode_step loop differs from selftok_decode"
    g_ms, s_ms = [], []
    for _ in range(3):
        g_ms.append(events_ms(lambda: eng.decode(tok, noise)))
        s_ms.append(events_ms(steps_loop))
    assert torch.equal(x, eng.decode(tok, noise))
    static_ips = B / (np.median(g_ms) / 1e3)
    out["homogeneous"] = {"decode_graph_ms": g_ms, "decode_step_x50_ms": s_ms, "ratio_median": float(np.median(s_ms) / np.median(g_ms)),
                          "bitwise_equal": True, "static_images_per_s": static_ips}
    print(json.dumps({"homogeneous": out["homogeneous"]}))

    # ---- 2. staggered steady state
    st = (np.arange(B) * T // B).astype(np.int32)              # rows spread over 0..T-1
    xs = noise.clone()

    def one_step():
        eng.decode_step(tok, xs, st, out=xs)
        st[:] += 1
        done = np.nonzero(st >= T)[0]
        if done.size:                                          # re-admitted at row 0 with fresh noise
            idx = torch.as_tensor(done, device=xs.device)
            xs.index_copy_(0, idx, noise.index_select(0, idx))
            st[done] = 0

    for _ in range(10):
        one_step()
    flops, n_steps = 0.0, T
    st_start = st.copy()
    for i in range(n_steps):
        flops += sum(step_flops[(int(s) + i) % T] for s in st_start)
    st[:] = st_start
    ms = events_ms(lambda: [one_step() for _ in range(n_steps)])
    step_ms = ms / n_steps
    ips = B / (T * step_ms / 1e3)
    out["staggered"] = {"steps": n_steps, "ms_total": ms, "step_ms": step_ms, "images_per_s": ips, "share_of_static": ips / static_ips,
                        "useful_tflop_per_s": flops / 1e12 / (ms / 1e3)}
    print(json.dumps({"staggered": out["staggered"]}))

    # ---- 3. arrival trace, real time
    host_tok = tok.cpu()
    host_noise = noise.cpu()
    t_batch = np.median(g_ms) / 1e3

    def run_continuous(rate):
        dec = ContinuousDecoder(eng, B)
        arrive = np.arange(a.requests) / rate
        lat, sent, t0 = {}, 0, time.perf_counter()
        t_arr = {}
        while len(lat) < a.requests:
            now = time.perf_counter() - t0
            while sent < a.requests and arrive[sent] <= now:
                rid = dec.submit(host_tok[sent % B], host_noise[sent % B:sent % B + 1])
                t_arr[rid] = arrive[sent]
                sent += 1
            if dec.active or dec.pending:
                res = dec.step()
                torch.cuda.synchronize()
                done_t = time.perf_counter() - t0
                for rid, _ in res:
                    lat[rid] = done_t - t_arr[rid]
            else:
                time.sleep(max(0.0, arrive[sent] - (time.perf_counter() - t0)))
        return np.array(list(lat.values())), time.perf_counter() - t0

    def run_static(rate):
        arrive = np.arange(a.requests) / rate
        lat, sent, queue, t0 = [], 0, [], time.perf_counter()
        buf_tok, buf_noise = tok.clone(), noise.clone()
        while len(lat) < a.requests:
            now = time.perf_counter() - t0
            while sent < a.requests and arrive[sent] <= now:
                queue.append(sent)
                sent += 1
            if queue and (len(queue) >= B or now - arrive[queue[0]] >= t_batch or sent == a.requests):
                take, queue = queue[:B], queue[B:]
                for j, r in enumerate(take):                   # padded to the captured B = 64 graph
                    buf_tok[j].copy_(tok[r % B])
                    buf_noise[j].copy_(noise[r % B])
                eng.decode(buf_tok, buf_noise)
                torch.cuda.synchronize()
                done_t = time.perf_counter() - t0
                lat += [done_t - arrive[r] for r in take]
            else:
                nxt = arrive[sent] if sent < a.requests else np.inf
                dl = arrive[queue[0]] + t_batch if queue else np.inf
                time.sleep(max(0.0, min(nxt, dl) - (time.perf_counter() - t0)))
        return np.array(lat), time.perf_counter() - t0

    out["arrivals"] = []
    for load in (0.5, 0.9):
        rate = load * static_ips
        for name, fn in (("continuous", run_continuous), ("static", run_static)):
            lat, wall = fn(rate)
            rec = {"policy": name, "load": load, "rate_per_s": rate, "requests": a.requests, "p50_s": float(np.percentile(lat, 50)),
                   "p95_s": float(np.percentile(lat, 95)), "completed_images_per_s": a.requests / wall}
            out["arrivals"].append(rec)
            print(json.dumps(rec))

    # ---- where a staggered step's time goes (separate run of the profiler)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            one_step()
        torch.cuda.synchronize()
    with open(os.path.join(a.out, "continuous_profile.txt"), "w") as f:
        f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25))
    out["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "continuous_bench.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({"gpu": out["gpu_after"]}))
    eng.close()


if __name__ == "__main__":
    main()
