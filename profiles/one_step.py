"""One sampler step (step 0: all 512 tokens visible, batch 64) with CUDA graphs off, for per-launch ncu lists:

    ncu --metrics gpu__time_duration.sum,sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active --clock-control none \
        -k regex:"gemm_tc|attention_tc|ln_mod" --csv --log-file step0_launches.csv python profiles/one_step.py
"""
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from selftoktokenizer_b200 import capi, config as C, synth  # noqa: E402

dev = torch.device("cuda:0")
d = C.FULL
prec = sys.argv[1] if len(sys.argv) > 1 else "fp16"
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 1
eng = capi.Engine(d, synth.synth_state_dict(d, device=dev), device=dev, precision=prec)
B = 64
tok = torch.randint(0, d.codebook_size, (B, d.K), device=dev)
noise = torch.randn(B, d.in_channels, d.latent, d.latent, device=dev)
eng.set_use_graph(False)
eng.decode(tok, noise, steps=steps)
torch.cuda.synchronize()
print("done", eng.last_launch_count)
