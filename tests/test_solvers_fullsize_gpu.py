"""Full-size parity of the DPM-Solver++(2M) step: 3 steps of the production loop at SDXL width and config-2 shapes (a
first-order step, then two second-order steps that read the x0_prev state the kernel carried), against the float64-rule
oracle loop (oracle/solver_ref.py) in fp32 (ref32) and under fp16 autocast with fp16 weights (ref16), gated by the policy
of tests/test_fullsize_gpu.py: engine vs ref32 <= ref16 vs ref32 + 2.5e-4."""
import pytest
import torch

from test_fullsize_gpu import _cast, _err, _forward_inputs, _gate, _record, full  # noqa: F401  (module-scoped fixture)

pytestmark = pytest.mark.gpu


def test_fullsize_dpmpp_2m_loop_vs_oracle(full):  # noqa: F811
    from oracle import solver_ref as SV
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.scheduler import DDPMScheduler, DPMSolverMultistepScheduler
    B, h, w, steps, run = 2, 128, 96, 20, 3
    inp = _forward_inputs(full["cfg_t"], full["cfg_g"], B, h, w, seed=3)
    sch = DPMSolverMultistepScheduler.from_config(DDPMScheduler().config)
    sch.set_timesteps(steps)
    den = TryOnDenoiser(full["eng_t"], full["eng_g"])
    den.prepare(**inp, guidance_scale=2.0)
    den.set_step_tables(sch, sch.timesteps)
    assert den.kind == "dpmpp" and [r[-1] > 0 for r in den.coef_table[:run].tolist()] == [False, True, True]
    for i in range(run):
        den.step(i, None, use_graph=True)
    torch.cuda.synchronize()
    lat = den.latents.clone()
    del den
    ts = sch.timesteps[:run]
    with torch.no_grad():
        ref = SV.denoise_loop(full["sd_t32"], full["cfg_t"], full["sd_g32"], full["cfg_g"], inp, sch, "dpmpp", ts)
        with torch.autocast("cuda", dtype=torch.float16):
            ref16 = SV.denoise_loop(full["sd_t"], full["cfg_t"], full["sd_g"], full["cfg_g"], _cast(inp, torch.float16),
                                    sch, "dpmpp", ts)
    d_eng32, d_ref32, d_eng16 = _err(lat, ref), _err(ref16, ref), _err(lat, ref16)
    _record(case=f"DPM-Solver++(2M) loop {run} of {steps} steps B={B} {h}x{w}", latents_absmax=ref.abs().max().item(),
            latents=dict(eng_vs_32=d_eng32, ref16_vs_32=d_ref32, eng_vs_ref16=d_eng16))
    _gate("latents (DPM-Solver++)", d_eng32, d_ref32, d_eng16)
