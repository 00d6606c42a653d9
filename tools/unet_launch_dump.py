#!/usr/bin/env python
"""Per-launch CUDA-event timing of one SD v1-4 U-Net call (batch 8 by default) with the GEMM shapes: run with
    CDX_PROF_DUMP=1 python tools/unet_launch_dump.py [batch] 2> unet_launches.txt"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from cycle_diffusion_b200 import specs  # noqa: E402
from cycle_diffusion_b200.engine import Engine, UNet  # noqa: E402

os.environ.setdefault('CDX_PROF_DUMP', '1')
B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
eng = Engine(0)
cfg = specs.sd_unet_config(768)
unet = UNet(eng, cfg, 'openai').load_state_dict(specs.synth_state_dict(specs.openai_unet_params(cfg), 1234))
x = torch.randn(B, 4, 64, 64, device='cuda')
t = torch.full((B,), 501., device='cuda')
ctx = torch.randn(B, 77, 768, device='cuda')
for _ in range(2):
    unet(x, t, ctx)
eng.profile(True)
unet(x, t, ctx)
fam = eng.profile_read()
eng.profile(False)
print({k: round(v['ms'], 3) for k, v in fam.items()})
