"""Profiler target (torch.cuda.profiler range): one fp32 VAE encoder pass of 6 images (masked image, pose, garment of a config-2 batch) and one
decoder pass of 2 latents at 1024x768, after one warm-up of each (profiler range around the measured passes)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import idm_vton_b200  # noqa: F401,E402
from idm_vton_b200.vae import AutoencoderKL  # noqa: E402

torch.manual_seed(0)
vae = AutoencoderKL().to("cuda", torch.float32).eval()
x = torch.rand(6, 3, 1024, 768, device="cuda") * 2 - 1
z = torch.randn(2, 4, 128, 96, device="cuda")
with torch.no_grad():
    for measured in (False, True):
        if measured:
            torch.cuda.synchronize()
            torch.cuda.cudart().cudaProfilerStart()
        vae.encode(x).latent_dist.mode()
        vae.decode(z, return_dict=False)
        torch.cuda.synchronize()
        if measured:
            torch.cuda.cudart().cudaProfilerStop()
