"""Profiler target (torch.cuda.profiler range): the CLIP ViT-H self-attention launch (B=2, 16 heads of 80, 257 tokens) and the bigG text one (B=2, 20 heads of
64, 77 tokens, causal), a few times each."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import idm_vton_b200  # noqa: F401,E402
from idm_vton_b200 import lib as L  # noqa: E402

L.load()
g = torch.Generator(device="cuda").manual_seed(0)
for (B, H, N, D, causal) in ((2, 16, 257, 80, False), (2, 20, 77, 64, True)):
    qkv = torch.randn(B, N, 3 * H * D, generator=g, device="cuda", dtype=torch.float16)
    C = H * D
    for _ in range(4):
        L.encoder_attention(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], H, D, causal=causal)
torch.cuda.synchronize()
