"""diffusers.image_processor for the shim: the reference pipeline only needs `VaeImageProcessor.preprocess/postprocess`
(src/tryon_pipeline.py:418-421,1588-1602,1885). diffusers is not installable here, so the restatement that ships with
the product (idm-vton_b200/vae.py, host-side plumbing) serves both sides; its semantics are "parity unpinned"
(no diffusers source under the reference)."""
import os
import sys

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)
from idm_vton_b200.vae import VaeImageProcessor  # noqa: E402,F401

PipelineImageInput = object
