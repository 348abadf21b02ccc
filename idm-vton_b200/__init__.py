"""idm-vton_b200 — Hopper-native (sm_90a) engine for IDM-VTON's denoising hot path.

Import as `idm_vton_b200` (the root-level `idm_vton_b200.py` maps the importable name onto this directory).
Layout: csrc/ (hand-written CUDA + C ABI), lib.py (ctypes binding), engine.py (UNet executors),
unet.py / pipeline.py (host-side mirrors of the reference's UNet2DConditionModel / StableDiffusionXLInpaintPipeline).
"""
__version__ = "0.1.0"
