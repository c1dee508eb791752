"""SD3 VAE decode / encode throughput on the device at several image sizes, and how much of each size's convolution tiles is
useful work.

    python profiles/vae_sizes.py [--reps 3] [--compare OTHER_LIB]

For every size: images/s of `selftok_vae_decode` (latents -> pixels, norm_ip) and `selftok_vae_encode` (pixels -> latent means),
CUDA events around 3 batches after one warm-up batch, and the output pixels the implicit-GEMM 3x3 convolutions execute
(whole 128-pixel tiles, some overhanging the image edge) against the pixels they keep, summed over one image's convolutions.
The batch holds 64 x 256 x 256 pixels (at most 64 images), so every size moves about the same data per batch.

--compare OTHER_LIB runs another build of libselftok_b200.so (e.g. the parent commit's) and this one alternately, `--reps` times
each, at 256 and 512, each run in its own process; it also checks that both builds give bitwise the same outputs for decode at
latent 8, 16, 32, 64 and encode at 128, 256, 512 on the same seeded inputs.  The card, its power limit and the SM clock are read
in the same run.  Nothing is written to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(96, 96), (192, 192), (256, 256), (384, 384), (512, 512), (640, 384)]
CH, MULT = 128, (1, 2, 4, 4)


# ---------------------------------------------------------------------------------------------- tile accounting (host only)
def conv_box(H, W, stride):
    """(bw, bh, bn) of the convolution A box, as gemm_tc.cu conv_box chooses it with conv_edge set."""
    hw = H * W
    exact = ((W % 128 == 0 or 128 % W == 0) and (hw % 128 == 0 or 128 % hw == 0)
             and (W >= 128 or hw < 128 or H % (128 // W) == 0) and (stride == 1 or hw % 128 == 0))
    if exact:
        bw = min(W, 128)
        bh = min(128 // bw, H)
        return bw, bh, 128 // (bw * bh)
    best = None
    bw = 128
    while bw >= 1:
        bh = 128 // bw
        n = -(-W // bw) * -(-H // bh)
        if best is None or n < best[0]:
            best = (n, bw, bh)
        bw //= 2
    return best[1], best[2], 1


def conv_dims(H, W, half):
    """(H, W, stride) of every 3x3 convolution of one image: `half` is "decode" (H, W = latent) or "encode" (H, W = image)."""
    out = []
    if half == "decode":
        out += [(H, W, 1)] * 5                                        # conv_in, mid.block_1 / 2
        h, w = H, W
        for lvl in (3, 2, 1, 0):
            out += [(h, w, 1)] * 6
            if lvl:
                h, w = 2 * h, 2 * w
                out.append((h, w, 1))                                 # upsample conv
        out.append((h, w, 1))                                         # conv_out
    else:
        out.append((H, W, 1))                                         # conv_in
        h, w = H, W
        for lvl in range(4):
            out += [(h, w, 1)] * 4
            if lvl != 3:
                h, w = h // 2, w // 2
                out.append((h, w, 2))                                 # downsample (output dims)
        out += [(h, w, 1)] * 5                                        # mid.block_1 / 2, conv_out
    return out


def tile_pixels(H, W, half):
    executed = useful = 0
    for h, w, s in conv_dims(H, W, half):
        bw, bh, bn = conv_box(h, w, s)
        executed += h * w if bn > 1 else -(-w // bw) * bw * -(-h // bh) * bh
        useful += h * w
    return executed, useful


def batch_for(H, W):
    return max(1, min(64, 64 * 256 * 256 // (H * W)))


# ---------------------------------------------------------------------------------------------- device runs (worker process)
def worker(sizes, dump):
    import numpy as np
    import torch
    sys.path.insert(0, REPO)
    from selftoktokenizer_b200 import synth
    from selftoktokenizer_b200.capi import VaeDecoder
    dev = torch.device("cuda:0")
    vae = VaeDecoder(synth.synth_vae_state_dict(ch=CH, device=dev), device=dev)
    if dump:
        out = {}
        for h in (8, 16, 32, 64):
            z = synth.synth_tensor(f"vae_sizes.cmp.z{h}", (2, 16, h, h), "emb", 1.0, device=dev)
            out[f"dec{h}"] = vae.decode(z).cpu().numpy()
        for H in (128, 256, 512):
            x = synth.synth_tensor(f"vae_sizes.cmp.x{H}", (2, 3, H, H), "emb", 0.5, device=dev)
            m, lv = vae.encode(x, return_logvar=True)
            out[f"enc{H}"] = torch.cat([m, lv], 1).cpu().numpy()
        np.savez(dump, **out)
    for H, W in sizes:
        B = batch_for(H, W)
        z = synth.synth_tensor("bench.noise.0", (B, 16, H // 8, W // 8), "emb", 0.5, device=dev)
        img = synth.synth_tensor("bench.images", (B, 3, H, W), "emb", 0.5, device=dev)
        rec = {"size": f"{H}x{W}", "batch": B}
        for name, fn in (("decode", lambda: vae.decode(z, norm_ip=True)), ("encode", lambda: vae.encode(img))):
            fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(3):
                fn()
            e1.record()
            torch.cuda.synchronize()
            rec[f"{name}_img_s"] = round(3 * B / (e0.elapsed_time(e1) / 1000.0), 2)
        print(json.dumps(rec), flush=True)
        torch.cuda.empty_cache()
    vae.close()


def run_worker(lib, sizes, dump=None):
    env = dict(os.environ)
    if lib:
        env["SELFTOK_B200_LIB"] = os.path.abspath(lib)
    cmd = [sys.executable, os.path.abspath(__file__), "--worker", json.dumps(sizes)] + (["--dump", dump] if dump else [])
    r = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"worker failed ({lib or 'this build'}):\n{r.stdout}\n{r.stderr[-3000:]}")
    return [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--compare", default=None, help="another libselftok_b200.so to alternate with this build at 256 / 512")
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--dump", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        worker([tuple(s) for s in json.loads(a.worker)], a.dump)
        return
    print(f"card (name, power limit, SM clock, max SM clock): {card()}")
    for H, W in SIZES:
        for half, (h, w) in (("decode", (H // 8, W // 8)), ("encode", (H, W))):
            ex, us = tile_pixels(h, w, half)
            print(f"{H}x{W} {half}: conv tiles execute {ex} output pixels per image for {us} useful ({us / ex:.3f})")
    result = {"card": None, "sizes": {}}
    if a.compare:
        with tempfile.TemporaryDirectory() as td:
            pa, pb = os.path.join(td, "other.npz"), os.path.join(td, "this.npz")
            run_worker(a.compare, [], pa)
            run_worker(None, [], pb)
            import numpy as np
            ga, gb = np.load(pa), np.load(pb)
            same = {k: bool(np.array_equal(ga[k].view(np.int32), gb[k].view(np.int32))) for k in ga.files}
            print(f"bitwise equal outputs, other build vs this build: {same}")
            result["bitwise_equal_to_other"] = all(same.values())
        runs = {"other": [], "this": []}
        for _ in range(a.reps):
            for tag, lib in (("other", a.compare), ("this", None)):
                for rec in run_worker(lib, [(256, 256), (512, 512)]):
                    runs[tag].append(rec)
                    print(f"[{tag}] {json.dumps(rec)}", flush=True)
        for tag, recs in runs.items():
            for size in ("256x256", "512x512"):
                for k in ("decode_img_s", "encode_img_s"):
                    v = [r[k] for r in recs if r["size"] == size]
                    print(f"{tag} {size} {k}: min {min(v):.1f} max {max(v):.1f} ({', '.join(f'{x:.1f}' for x in v)})")
        result["compare"] = runs
    for rec in run_worker(None, SIZES):
        H, W = (int(x) for x in rec["size"].split("x"))
        ex_d, us_d = tile_pixels(H // 8, W // 8, "decode")
        ex_e, us_e = tile_pixels(H, W, "encode")
        rec.update(decode_tile_pixels=[ex_d, us_d], encode_tile_pixels=[ex_e, us_e])
        result["sizes"][rec.pop("size")] = rec
    result["card"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
