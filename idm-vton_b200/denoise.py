"""The denoising hot loop of IDM-VTON on the engine (src/tryon_pipeline.py:1765-1866).

Per step the reference runs the garment UNet (batch Bg), zero-pads its 70 features for the CFG-uncond half, runs the
try-on UNet (batch 2B), applies CFG and the DDPM update. Here one step is a fixed launch sequence over static buffers:
  latents -> [NCHW->NHWC scatter into the 13(+pad)-channel input] -> garment UNet -> try-on UNet (garment K/V streamed
  as a second attention segment, uncond half in closed form) -> fused CFG(+guidance rescale)+DDPM, or fused CFG +
  DDIM / Euler / DPM-Solver++ step (Euler scales the latents in the scatter)
captured once in a CUDA graph and replayed per step; step-invariant work (cross-attention K/V of text / IP tokens,
aug_emb, the static input channels) is hoisted to prepare().
"""
import collections

import torch

from .engine import CIN_PAD, UNetEngine
from .lib import KV8_GROUP, GarmentKV8
from .scheduler import DPMSolverMultistepScheduler, _init_step_index, config_getter, solver_order_at


class nvtx_range:
    """NVTX range around a host-side stage (visible in nsys / ncu --nvtx; a no-op cost of ~1 us otherwise)."""

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        torch.cuda.nvtx.range_push(self.name)

    def __exit__(self, *a):
        torch.cuda.nvtx.range_pop()


_KINDS = {"DDPMScheduler": "ddpm", "DDIMScheduler": "ddim", "EulerDiscreteScheduler": "euler",
          "DPMSolverMultistepScheduler": "dpmpp"}


def scheduler_kind(scheduler):
    """"ddpm" | "ddim" | "euler" | "dpmpp": the fused step that implements `scheduler`, from the class names of its
    type (so a caller's own diffusers scheduler, or a subclass of one, is recognised). An object whose class is not a
    `...Scheduler` (a bare object carrying the DDPM attributes) is treated as DDPM; every other scheduler class
    raises NotImplementedError instead of being stepped with the wrong update."""
    for c in type(scheduler).__mro__:
        if c.__name__ in _KINDS:
            return _KINDS[c.__name__]
    name = type(scheduler).__name__
    if name.endswith("Scheduler"):
        raise NotImplementedError(
            f"{name} is not supported by the engine: its fused step implements DDPMScheduler, DDIMScheduler, "
            "EulerDiscreteScheduler (s_churn = 0) and DPMSolverMultistepScheduler (dpmsolver++, midpoint, order <= 2)")
    return "ddpm"


def check_guidance_rescale(scheduler, guidance_rescale):
    """Refuses guidance_rescale > 0 with any step but DDPM's: the guidance rescale is fused with the DDPM step only."""
    if guidance_rescale > 0 and scheduler_kind(scheduler) != "ddpm":
        raise NotImplementedError(f"guidance_rescale with {type(scheduler).__name__}: the engine's guidance rescale is "
                                  "fused with the DDPM step only")


def ddim_step_coefficients(scheduler, t, eta=0.0):
    """(s, inv_a, p, q, r, sigma_n, k) of DDIMScheduler.step at timestep t (the coefficient layout of
    b200vton_cfg_solver_step), computed in fp32 torch like diffusers 0.25 from the generic attributes:
    `alphas_cumprod`, `final_alpha_cumprod` (or `config.set_alpha_to_one`), `config.num_train_timesteps` and
    `num_inference_steps`. The step goes to t - T_train // num_inference_steps."""
    get = config_getter(getattr(scheduler, "config", None))
    if get("prediction_type", "epsilon") != "epsilon" or get("clip_sample", False) or get("thresholding", False):
        raise NotImplementedError("the fused DDIM step covers epsilon prediction without clip_sample / thresholding")
    ac = scheduler.alphas_cumprod.to(device="cpu", dtype=torch.float32)
    t = int(t)
    prev_t = t - int(get("num_train_timesteps", len(ac))) // int(scheduler.num_inference_steps)
    final = getattr(scheduler, "final_alpha_cumprod", None)
    if final is None:
        final = torch.tensor(1.0) if get("set_alpha_to_one", True) else ac[0]
    a_t = ac[t]
    a_prev = ac[prev_t] if prev_t >= 0 else torch.as_tensor(final, dtype=torch.float32).cpu()
    var = (1 - a_prev) / (1 - a_t) * (1 - a_t / a_prev)
    std = eta * var ** 0.5
    inv_a = torch.tensor(1.0, dtype=torch.float32) / (a_t ** 0.5)
    return (float((1 - a_t) ** 0.5), float(inv_a), 0.0, float(a_prev ** 0.5), float((1 - a_prev - std ** 2) ** 0.5),
            float(std), 0.0)


def _run_indices(scheduler, timesteps):
    """Positions in `scheduler.timesteps` of the timesteps a run steps through: the first found like diffusers'
    `_init_step_index` (the second match when it occurs twice), then one further per step."""
    sched = scheduler.timesteps.detach().cpu().to(torch.float64)
    run = [float(t) for t in timesteps]
    start = _init_step_index(sched, run[0])
    if sched[start:start + len(run)].tolist() != run:
        raise ValueError("the run's timesteps must be consecutive entries of the scheduler's timesteps")
    return list(range(start, start + len(run)))


def euler_step_tables(scheduler, timesteps):
    """([(s, inv_a, p, q, r, sigma_n, k)], [input scale]) per step of EulerDiscreteScheduler at s_churn = 0 (the
    pipeline passes no s_churn), in fp32 torch like diffusers 0.25, from `sigmas` (N + 1 values) and `timesteps`."""
    get = config_getter(getattr(scheduler, "config", None))
    if get("prediction_type", "epsilon") != "epsilon" or get("interpolation_type", "linear") != "linear":
        raise NotImplementedError("the fused Euler step covers epsilon prediction with linear sigma interpolation")
    sig = scheduler.sigmas.detach().to(device="cpu", dtype=torch.float32)
    rows, scales = [], []
    for i in _run_indices(scheduler, timesteps):
        sigma, sigma_next = sig[i], sig[i + 1]
        rows.append((float(sigma), float(torch.tensor(1.0) / sigma), 1.0, 0.0, float(sigma_next - sigma), 0.0, 0.0))
        scales.append(float(torch.tensor(1.0) / ((sigma ** 2 + 1) ** 0.5)))
    return rows, scales


def dpmpp_step_coefficients_table(scheduler, timesteps):
    """[(s, inv_a, p, q, r, sigma_n, k)] per step of DPMSolverMultistepScheduler (dpmsolver++, midpoint, order 1 / 2),
    in fp32 torch like diffusers 0.25, from `sigmas`, `timesteps` and the config's solver_order, lower_order_final and
    euler_at_final; k = 1 / r0 at second-order steps and 0 at first-order ones."""
    get = config_getter(getattr(scheduler, "config", None))
    if get("solver_order", 2) not in (1, 2):
        raise NotImplementedError(f"solver_order {get('solver_order')}: the fused DPM-Solver++ step covers orders 1 and 2")
    if get("algorithm_type", "dpmsolver++") != "dpmsolver++":
        raise NotImplementedError(f"algorithm_type {get('algorithm_type')}: the fused step covers dpmsolver++ only")
    if get("solver_type", "midpoint") != "midpoint":
        raise NotImplementedError(f"solver_type {get('solver_type')}: the fused step covers midpoint only")
    if get("thresholding", False) or get("prediction_type", "epsilon") != "epsilon" or get("use_lu_lambdas", False):
        raise NotImplementedError("the fused DPM-Solver++ step covers epsilon prediction without thresholding or "
                                  "use_lu_lambdas")
    sig = scheduler.sigmas.detach().to(device="cpu", dtype=torch.float32)
    n = len(scheduler.timesteps)
    alpha_sigma = DPMSolverMultistepScheduler._sigma_to_alpha_sigma_t
    rows = []
    for j, i in enumerate(_run_indices(scheduler, timesteps)):
        alpha_t, sigma_t = alpha_sigma(sig[i])
        alpha_n, sigma_n = alpha_sigma(sig[i + 1])
        lam = torch.log(alpha_t) - torch.log(sigma_t)
        h = torch.log(alpha_n) - torch.log(sigma_n) - lam
        c = alpha_n * (torch.exp(-h) - 1.0)
        k = 0.0
        if solver_order_at(j, i, n, scheduler.config) == 2:
            alpha_p, sigma_p = alpha_sigma(sig[i - 1])
            r0 = (lam - (torch.log(alpha_p) - torch.log(sigma_p))) / h
            k = float(1.0 / r0)
        rows.append((float(sigma_t), float(torch.tensor(1.0) / alpha_t), float(sigma_n / sigma_t), float(-c), 0.0, 0.0, k))
    return rows


def solver_step_tables(scheduler, timesteps, eta=0.0):
    """The per-step tables of the fused step for `scheduler` over the run's `timesteps`:
    (kind, rows, scales, draws, noise_applied). rows: the kernel's coefficients after the guidance scale (5 DDPM values
    for "ddpm", the 7 of b200vton_cfg_solver_step otherwise); scales: the input scale of each step (Euler's
    scale_model_input, else None); draws: whether the scheduler's own `step` draws a variance-noise tensor from the
    generator at that step (DDPM at t > 0, DDIM at eta > 0, Euler at every step); noise_applied: whether that draw enters
    the update (Euler draws it and multiplies it by zero at s_churn = 0)."""
    kind = scheduler_kind(scheduler)
    T = len(timesteps)
    if kind == "ddpm":
        return kind, [ddpm_step_coefficients(scheduler, int(t)) for t in timesteps], None, \
            [int(t) > 0 for t in timesteps], True
    if kind == "ddim":
        return kind, [ddim_step_coefficients(scheduler, t, eta) for t in timesteps], None, [eta > 0] * T, True
    if kind == "euler":
        rows, scales = euler_step_tables(scheduler, timesteps)
        return kind, rows, scales, [True] * T, False
    return kind, dpmpp_step_coefficients_table(scheduler, timesteps), None, [False] * T, False


def ddpm_step_coefficients(scheduler, t):
    """(sqrt(1-abar_t), 1/sqrt(abar_t), x0 coeff, x_t coeff, sigma_t) of DDPMScheduler.step at timestep t, computed in
    fp32 torch like diffusers does, from the GENERIC scheduler interface only — `alphas_cumprod`,
    `config.num_train_timesteps`, `num_inference_steps` (and `previous_timestep` when the object has it) — so the
    caller's own `diffusers.DDPMScheduler` works (inference.py passes `DDPMScheduler.from_pretrained(...)`). The fused
    kernel implements epsilon prediction with fixed_small variance and no clipping / thresholding: anything else raises.
    A custom timestep list (`custom_timesteps`) needs `previous_timestep`: the even spacing t - T_train // steps would
    be wrong for it."""
    get = config_getter(getattr(scheduler, "config", None))
    if get("prediction_type", "epsilon") != "epsilon" or get("variance_type", "fixed_small") != "fixed_small" \
            or get("clip_sample", False) or get("thresholding", False):
        raise NotImplementedError("the fused CFG+DDPM step covers epsilon prediction, fixed_small variance, no "
                                  "clip_sample / thresholding (the IDM-VTON scheduler config)")
    if not hasattr(scheduler, "alphas_cumprod"):
        raise TypeError(f"{type(scheduler).__name__} has no alphas_cumprod: the engine needs a DDPM-family scheduler")
    t = int(t)
    n_train = int(get("num_train_timesteps", len(scheduler.alphas_cumprod)))
    if hasattr(scheduler, "previous_timestep"):
        prev_t = int(scheduler.previous_timestep(t))
    elif getattr(scheduler, "custom_timesteps", False):
        raise TypeError(f"{type(scheduler).__name__} has a custom timestep list but no previous_timestep(): the step "
                        "from each timestep to the next cannot be derived")
    else:
        steps = getattr(scheduler, "num_inference_steps", None) or n_train
        prev_t = t - n_train // steps
    ac = scheduler.alphas_cumprod.to(device="cpu", dtype=torch.float32)
    a_t = ac[t]
    a_prev = ac[prev_t] if prev_t >= 0 else torch.tensor(1.0)
    b_t, b_prev = 1 - a_t, 1 - a_prev
    cur_a = a_t / a_prev
    cur_b = 1 - cur_a
    c0 = (a_prev ** 0.5 * cur_b) / b_t
    c1 = cur_a ** 0.5 * b_prev / b_t
    var = torch.clamp((1 - a_prev) / (1 - a_t) * cur_b, min=1e-20)
    sigma = var ** 0.5 if t > 0 else torch.tensor(0.0)
    inv_sa = torch.tensor(1.0, dtype=torch.float32) / (a_t ** 0.5)
    return float(b_t ** 0.5), float(inv_sa), float(c0), float(c1), float(sigma)


MIXED_KIND_CODES = {"ddim": 0, "euler": 1, "dpmpp": 2, "ddpm": 3}     # kinds[b] of b200vton_cfg_step_mixed_rows


def identity_step_row(kind):
    """The coefficient row of an idle slot of SlotDenoiser: the step returns its latents unchanged (zeros stay zeros),
    whatever the finite eps. DDPM {gs, sb, inv_sa, c0, c1, sigma, phi, 0}: x0 = 0, prev = 1 * x; DDIM and DPM-Solver++
    {gs, s, inv_a, p, q, r, sigma_n, k}: x0 = x, out = fp16(1 * x0) (DDIM) or 1 * x + fp16(0 * x0) (DPM++); Euler:
    x0 = x - 0, d = 0, out = x + 0."""
    return {"ddpm": [0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0],
            "ddim": [0.0, 0.0, 1.0, 0.0, 1.0, 0.0, 0.0, 0.0],
            "euler": [0.0] * 8,
            "dpmpp": [0.0, 0.0, 1.0, 1.0, 0.0, 0.0, 0.0, 0.0]}[kind]


class StepPlan(collections.namedtuple("StepPlan", "kind coef_table t_table scale_table step_draws noise_applied T")):
    """The per-step tables of one run (step_plan), in the layout the step kernels read. coef_table [T + 1, 8] fp32: row
    i = the coefficients of step i, {gs, sb, inv_sa, c0, c1, sigma, phi, 0} for DDPM and {gs, s, inv_a, p, q, r,
    sigma_n, k} of b200vton_cfg_solver_step otherwise; row T = the idle row (identity_step_row). t_table [T + 1] fp32:
    the timesteps (fractional for Euler's linspace spacing), 0 at row T. scale_table [T + 1] fp32: Euler's input
    scales, 1 at row T; None for the other kinds. step_draws, noise_applied: as solver_step_tables. T: steps in the run."""

    def to(self, device):
        return self._replace(coef_table=self.coef_table.to(device), t_table=self.t_table.to(device),
                             scale_table=None if self.scale_table is None else self.scale_table.to(device))


def step_plan(scheduler, timesteps, guidance_scale, guidance_rescale=0.0, eta=0.0):
    """The StepPlan of a run of `scheduler` over `timesteps` (solver_step_tables, with DDIM's `eta`) at guidance scale gs
    and guidance rescale phi (DDPM only: check_guidance_rescale)."""
    check_guidance_rescale(scheduler, guidance_rescale)
    kind, coefs, scales, draws, applied = solver_step_tables(scheduler, timesteps, eta)
    gs = float(guidance_scale)
    rows = [[gs, *c, float(guidance_rescale), 0.0] if kind == "ddpm" else [gs, *c] for c in coefs]
    f32 = torch.float32
    return StepPlan(kind, torch.tensor(rows + [identity_step_row(kind)], dtype=f32),
                    torch.tensor([float(t) for t in timesteps] + [0.0], dtype=f32),
                    None if scales is None else torch.tensor(list(scales) + [1.0], dtype=f32), draws, applied, len(coefs))


def variance_noise(den, i, shape, generator, device, dtype):
    """The variance noise of step i for a denoiser's `step`, or None. It is drawn from `generator` when the scheduler's own
    `step` would draw it (DDPM at t > 0, DDIM at eta > 0, Euler at every step: den.step_draws), so the generator ends
    in the reference's state, and dropped when the update does not apply it (Euler's: den.noise_applied)."""
    from .pipeline import randn_tensor
    noise = randn_tensor(shape, generator=generator, device=device, dtype=dtype) if den.step_draws[i] else None
    return noise if den.noise_applied else None


def garment_tokens(tryon, hg, wg):
    """Ng of every try-on block, in tryon.blocks() order: the garment's tokens at the block's level for a garment latent
    of hg x wg (the stride-2 convolutions round up)."""
    n, lvl_tokens = (hg, wg), {}
    for c in tryon.ch:
        lvl_tokens[c] = n[0] * n[1]
        n = ((n[0] - 1) // 2 + 1, (n[1] - 1) // 2 + 1)
    return [lvl_tokens[b.c] for b in tryon.blocks()]


def garment_kv_format(tryon):
    """"fp16" or "fp8": the format the denoisers hold the try-on engine's hoisted garment K/V in (UNetEngine.
    garment_kv_format; fp16 for an engine that names none)."""
    return getattr(tryon, "garment_kv_format", "fp16")


def freeu_setting(tryon):
    """(s1, s2, b1, b2) when the try-on engine runs FreeU in its forward (UNetEngine.freeu_active), else None."""
    active = getattr(tryon, "freeu_active", None)
    return None if active is None else active()


def new_garment_kv(tryon, rows, ng, blk, device=None):
    """Storage for `rows` rows of one try-on block's hoisted garment K/V in garment_kv_format(tryon): fp16
    [rows, Ng, 2C], or a GarmentKV8. device: the engine's by default (the host tier passes "cpu")."""
    device = tryon.device if device is None else device
    if garment_kv_format(tryon) == "fp8":
        return GarmentKV8.empty(rows, ng, blk.c, device)
    return torch.empty((rows, ng, 2 * blk.c), dtype=torch.float16, device=device)


def garment_kv_bytes_per_step(tryon, hg, wg, fmt=None):
    """Bytes of the hoisted K/V of ONE garment for one denoise step: sum over the try-on blocks of Ng * 2C fp16, or in
    the "fp8" format (default: the engine's garment_kv_format) Ng * 2C e4m3 plus 2C / 64 int8 exponents per token
    (Ng rounded up to 16)."""
    fmt = fmt or garment_kv_format(tryon)
    if fmt == "fp8":
        return sum(ng * 2 * b.c + (2 * b.c // KV8_GROUP) * (-(-ng // 16) * 16)
                   for b, ng in zip(tryon.blocks(), garment_tokens(tryon, hg, wg)))
    return sum(ng * 2 * b.c * 2 for b, ng in zip(tryon.blocks(), garment_tokens(tryon, hg, wg)))


def check_garment_kv_held(tryon, what):
    """FP8 garment K/V exist only as hoisted K/V: refuses, before any launch, a path that computes them in the step."""
    if garment_kv_format(tryon) != "fp8":
        return
    for name in ("b200vton_quantize_kv_e4m3", "b200vton_attention_kv8"):
        if not tryon.L.has_symbol(name):
            raise NotImplementedError(f"FP8 garment K/V need {name}, which this library binding does not export")
    if what is not None:
        raise NotImplementedError(f"garment K/V precision 'fp8' with {what}: only hoisted garment K/V are held in the "
                                  "FP8 format (the garment K/V of this path are computed inside the step)")


def kv_map(kv, fn):
    """fn applied to a block's hoisted garment K/V: the fp16 tensor, or both parts of a GarmentKV8 (rows first)."""
    return kv.map(fn) if isinstance(kv, GarmentKV8) else fn(kv)


def kv_parts(kv):
    return tuple(kv) if isinstance(kv, GarmentKV8) else (kv,)


def copy_kv_rows(dst, d0, src, s0, n=1):
    """dst[d0:d0 + n] = src[s0:s0 + n] for one block's hoisted garment K/V (the fp16 tensor, or the e4m3 rows and the
    int8 exponents of a GarmentKV8), enqueued on the current stream: one cudaMemcpyAsync per part, the rows being
    contiguous. Between page-locked host memory and the device the host does not wait for it. Returns the bytes."""
    nbytes = 0
    for d, s in zip(kv_parts(dst), kv_parts(src)):
        rows = s[s0:s0 + n]
        d[d0:d0 + n].copy_(rows, non_blocking=True)
        nbytes += rows.numel() * rows.element_size()
    return nbytes


def _host_register(t):
    """Page-locks the storage of CPU tensor t (cudaHostRegister); False when CUDA refuses."""
    return int(torch.cuda.cudart().cudaHostRegister(t.data_ptr(), t.numel() * t.element_size(), 0)) == 0


def _host_unregister(t):
    torch.cuda.cudart().cudaHostUnregister(t.data_ptr())


class HostGarmentKV:
    """Q pages of hoisted garment K/V in page-locked host memory, in the format of the device pool: per try-on block one
    fp16 [Q*T_page, Ng, 2C] tensor, or a GarmentKV8 of Q*T_page rows (e4m3 rows and int8 exponents); page q = rows
    q*T_page .. q*T_page + T_page - 1. The tensors are plain CPU tensors page-locked with cudaHostRegister: torch's
    pin_memory goes through its caching host allocator, which rounds every allocation up to a power of two (a 9.44 GB
    page could pin 16 GB). There is no pageable fallback: a failed allocation raises RuntimeError naming the bytes.
    release() unregisters them; it must come before the tensors are dropped."""

    def __init__(self, tryon, pages, T_page, h, w):
        self.Q, self.T_page = int(pages), int(T_page)
        self.bytes = self.Q * self.T_page * garment_kv_bytes_per_step(tryon, h, w)
        self.blocks, self._locked = [], []
        try:
            for b, ng in zip(tryon.blocks(), garment_tokens(tryon, h, w)):
                kv = new_garment_kv(tryon, self.Q * self.T_page, ng, b, device="cpu")
                for t in kv_parts(kv):
                    if not _host_register(t):
                        raise RuntimeError(f"cudaHostRegister refused {t.numel() * t.element_size()} bytes")
                    self._locked.append(t)
                self.blocks.append(kv)
        except (RuntimeError, MemoryError) as exc:
            self.release()
            raise RuntimeError(f"the garment K/V host tier could not allocate and page-lock {self.bytes} bytes "
                               f"({self.Q} pages of {self.bytes // self.Q} bytes) of host memory: {exc}") from exc

    def release(self):
        """Unregisters every page-locked tensor (idempotent); the tier holds nothing afterwards."""
        while self._locked:
            _host_unregister(self._locked.pop())
        self.blocks = []

    def __del__(self):
        try:
            self.release()
        except Exception:       # interpreter shutdown: CUDA may be gone, and the process releases everything
            pass


def hoisted_garment_kv(tryon, garment, x_g, ctx_g, t_table, t0, t1, chunk, out):
    """The hoisted garment passes of the timesteps t_table[t0:t1] for the Bg garments of x_g [Bg,hg,wg,64] / ctx_g
    (garment.encode_context of their text embeddings): the garment UNet batched over `chunk` timesteps per pass (large-M
    GEMMs, weights read once per chunk), then the garment K/V projection of every try-on block. out[i]: a contiguous
    [(t1 - t0) * Bg, Ng, 2C] view that receives block i's K/V in timestep-major order (row (t - t0) * Bg + g). The
    bits depend only on the garments, the timesteps and the chunking."""
    Bg = x_g.shape[0]
    blocks = tryon.blocks()
    T = t1 - t0
    for c0 in range(0, T, chunk):
        n = min(chunk, T - c0)
        t_rows = t_table[t0 + c0:t0 + c0 + n].repeat_interleave(Bg).contiguous()   # timestep-major rows
        x_big = x_g.repeat(n, 1, 1, 1)
        ctx_big = [(kv_t.repeat(n, 1, 1), None) for kv_t, _ in ctx_g]
        feats = []
        garment.forward(x_big, garment.time_embedding(t_rows, n * Bg), ctx_big, collect=feats)
        for i, (blk, f) in enumerate(zip(blocks, feats)):
            tryon.garment_kv(blk, f, out=kv_map(out[i], lambda t: t[c0 * Bg:(c0 + n) * Bg]))
        del feats, x_big, ctx_big
    tryon.release_kv_scratch()


def default_garment_chunk(Bg):
    """Timesteps per hoisted garment pass: B200VTON_GARMENT_CHUNK when set, else as many as keep a pass at <= 64
    samples."""
    return int(__import__("os").environ.get("B200VTON_GARMENT_CHUNK", "0")) or max(1, 64 // max(1, Bg))


class GarmentKVCache:
    """LRU cache of hoisted garment K/V across requests (SURVEY.md 8f item 4). One entry = the K/V of ONE garment for every
    denoise step and every try-on block ([T, Ng, 2C] fp16 per block: 9.44 GB of K and V at 768x1024 / 30 steps, computed
    from the shapes; a GarmentKV8 per block in the "fp8" format, 4.79 GB), keyed by the caller's garment id plus
    everything the values depend on (timestep list, the garment's latent size, the format). A hit replaces the
    garment's T garment-UNet passes by device-to-device copies (~2 ms)."""

    def __init__(self, max_bytes=16 << 30):   # beside 11 GB of weights and the step's K/V on an 80 GB H100
        self.max_bytes = int(max_bytes)
        self.entries = collections.OrderedDict()
        self.bytes = 0
        self.hits = self.misses = 0

    def get(self, key):
        e = self.entries.get(key)
        if e is None:
            self.misses += 1
            return None
        self.entries.move_to_end(key)
        self.hits += 1
        return e[0]

    def put(self, key, tensors):
        n = sum(p.numel() * p.element_size() for t in tensors for p in kv_parts(t))
        if n > self.max_bytes:
            return
        if key in self.entries:
            self.bytes -= self.entries.pop(key)[1]
        while self.entries and self.bytes + n > self.max_bytes:
            self.bytes -= self.entries.popitem(last=False)[1][1]
        self.entries[key] = (tensors, n)
        self.bytes += n

    def clear(self):
        """Drops every entry (the pipeline's UNet arithmetic changed: cached K/V would no longer be what it computes)."""
        self.entries.clear()
        self.bytes = 0


def _describe(x):
    """(address, shape, dtype) of a tensor, element-wise through the lists and tuples that hold per-block buffers."""
    if isinstance(x, torch.Tensor):
        return x.data_ptr(), x.shape, x.dtype
    if isinstance(x, (list, tuple)):
        return tuple(_describe(v) for v in x)
    return x


class _CapturedStep:
    """The step of the module docstring over static buffers, launched eagerly or replayed from a CUDA graph, as
    TryOnDenoiser and SlotDenoiser share it. Subclasses supply the garment K/V the try-on UNet reads (_gkv_pre; None:
    the garment UNet runs in the step) and the per-step uploads (_upload). ROWS: one coefficient row per sample."""

    ROWS = False
    # Programmatic dependent launch INSIDE the captured step only (B200VTON_PDL_GRAPH, default below): every kernel node
    # of the graph is one of this library's kernels, which call griddepcontrol.wait before they touch global
    # memory, so the set-up of kernel n+1 overlaps the tail of kernel n. Eager launches, which interleave with cuBLAS /
    # cuDNN / ATen kernels in the pipeline call, keep plain stream order unless B200VTON_PDL=1 asks otherwise.
    # Default: ON inside the graph, OFF for eager launches.
    PDL_IN_GRAPH = __import__("os").environ.get("B200VTON_PDL_GRAPH", "1") == "1"
    _graph = _graph_sig = None   # the captured step and the _signature it was captured at
    kinds = None                 # per-sample kind codes of the mixed-kind step (SlotDenoiser.configure_presets)

    def _signature(self):
        """What a captured step bakes in: the kernel selection, the try-on UNet's FreeU values, and the address, shape and
        dtype of every buffer the graph reads or writes (not of those it allocates while capturing, such as eps)."""
        gkv_pre = self._gkv_pre()
        garment = (self.x_g, self.t_g, self.ctx_g) if gkv_pre is None else gkv_pre
        return (self.kind, self.rescale, self.do_cfg, gkv_pre is not None, freeu_setting(self.tryon)) + _describe(
            [self.latents, self.latents_next, self.noise, self.x0_prev, self.x_t, self.t_t, self.coef, self.scale,
             self.kinds, self.aug, self.ctx_t, garment])

    def _launch_step(self):
        """The launch sequence of one denoise step over the static buffers (graph-capturable)."""
        L = self.L
        if self.kind in ("euler", "mixed"):                       # scale_model_input on the latent channels only
            scatter = L.nchw_to_nhwc_scaled_rows if self.ROWS else L.nchw_to_nhwc_scaled
            scatter(self.latents, self.x_t, self.scale, c_off=0)
        else:
            L.nchw_to_nhwc(self.latents, self.x_t, c_off=0)      # CFG duplication + channel concat as offsets
        gkv_pre, feats = self._gkv_pre(), None
        if gkv_pre is None:
            feats = []
            self.garment.forward(self.x_g, self.garment.time_embedding(self.t_g, self.x_g.shape[0]), self.ctx_g,
                                 collect=feats)
        temb_t = self.tryon.time_embedding(self.t_t, self.Bt, self.aug)
        self.eps = self.tryon.forward(self.x_t, temb_t, self.ctx_t, gfeats=feats, gkv_pre=gkv_pre,
                                      n_persons=self.latents.shape[0] if self.do_cfg else 0)
        if self.kind == "mixed":                                  # one kind per sample
            L.cfg_step_mixed_rows(self.eps, self.latents, self.noise, self.coef, self.kinds, self.x0_prev,
                                  do_cfg=self.do_cfg, out=self.latents_next)
        elif self.kind == "ddpm":
            step = L.cfg_ddpm_step_rows if self.ROWS else L.cfg_rescale_ddpm_step if self.rescale else L.cfg_ddpm_step
            step(self.eps, self.latents, self.noise, self.coef, do_cfg=self.do_cfg, out=self.latents_next)
        else:
            step = L.cfg_solver_step_rows if self.ROWS else L.cfg_solver_step
            step(self.eps, self.latents, self.noise if self.kind == "ddim" else None, self.coef, self.kind,
                 x0_prev=self.x0_prev, do_cfg=self.do_cfg, out=self.latents_next)
        self.latents.copy_(self.latents_next)

    def capture(self):
        """Capture one step into a CUDA graph (one warm-up launch on a side stream, then one recorded pass)."""
        self._graph = self._graph_sig = None                      # the old graph's memory goes before the new one's
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream())
        keep = self.latents.clone()
        keep_x0 = self.x0_prev.clone() if self.x0_prev is not None else None  # the warm-up step advances the state
        with torch.cuda.stream(s):
            self._launch_step()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        pdl_before = self.L.get_option("programmatic_launch", 0)
        if self.PDL_IN_GRAPH:
            self.L.set_option("programmatic_launch", 1)
        try:
            with torch.cuda.graph(g):
                self._launch_step()
        finally:
            if self.PDL_IN_GRAPH:
                self.L.set_option("programmatic_launch", pdl_before)
        self.latents.copy_(keep)
        if keep_x0 is not None:
            self.x0_prev.copy_(keep_x0)
        self._graph, self._graph_sig = g, self._signature()

    def _run(self, use_graph, name, *rows):
        """One step: _upload(*rows), then a replay of the graph (re-captured if its _signature changed) or the eager
        launches. The signature is read first: an upload may wait for the device, and this overlaps the running step."""
        stale = use_graph and self._graph_sig != self._signature()
        self._upload(*rows)
        with nvtx_range(name):
            if stale:
                self.capture()
            if use_graph:
                self._graph.replay()
            else:
                self._launch_step()
        return self.latents


class TryOnDenoiser(_CapturedStep):
    def __init__(self, tryon: UNetEngine, garment: UNetEngine, hoist_garment=True, garment_chunk=None, max_kv_bytes=None):
        """max_kv_bytes: budget for the resident garment K/V of the hoisted passes (default: 60% of the free device memory
        when the step tables are set). When all denoise steps do not fit (e.g. 1024x1024, 50 steps, batch 4 = 84 GB),
        the steps are hoisted window by window: K/V of `window` consecutive steps are resident at a time and the next
        window's garment passes run when the loop reaches it — same arithmetic, same graph.
        hoist_garment: the garment UNet depends on the timestep but not on the latents (SURVEY.md App. D.4), so all
        its passes are run BEFORE the loop, batched over `garment_chunk` timesteps at a time (large-M GEMMs, weights
        read once per chunk instead of once per step), and the garment K/V of every try-on block are projected once
        for all steps; the per-step graph then contains the try-on UNet only and walks the K/V by a device-side
        step index. Exactly the same arithmetic per (step, garment) as the step-by-step order."""
        self.tryon = tryon
        self.garment = garment
        self.L = tryon.L
        self.device = tryon.device
        self.hoist_garment = hoist_garment
        if garment_chunk is None:
            garment_chunk = int(__import__("os").environ.get("B200VTON_GARMENT_CHUNK", "0")) or None
        self._garment_chunk = garment_chunk      # None: as many timesteps per pass as keep the pass at <= 64 samples
        self.max_kv_bytes = max_kv_bytes
        self.gkv_all = None
        self.window = None
        self.win_start = -1

    # -------------------------------------------------------------------------------------------
    def prepare(self, latents, mask, masked_image_latents, pose_latents, cloth_latents, prompt_embeds,
                add_text_embeds, add_time_ids, image_embeds, text_embeds_cloth, guidance_scale=2.0, do_cfg=True,
                guidance_rescale=0.0):
        """guidance_rescale: phi of rescale_noise_cfg (src/tryon_pipeline.py:101-113), applied only under CFG; 0 keeps
        the plain CFG+DDPM kernel. All tensors on the device. latents [B,4,h,w]; mask [Bt,1,h,w], masked_image_latents / pose_latents
        [Bt,4,h,w], prompt_embeds [Bt,77,X], add_text_embeds [Bt,P], add_time_ids [Bt,6], image_embeds [Bt,16,X]
        with Bt = 2B under CFG ([uncond ; cond] order, src/tryon_pipeline.py:1711-1714); cloth_latents [Bg,4,hg,wg],
        text_embeds_cloth [Bg,77,X]. The garment may have a latent size of its own: the garment UNet runs at the cloth's
        size (src/tryon_pipeline.py:1654,1787) and its Ng tokens per level join the try-on attention as they are."""
        with nvtx_range("b200vton.prepare(context K/V, aug_emb, static input channels)"):
            self._prepare(latents, mask, masked_image_latents, pose_latents, cloth_latents, prompt_embeds, add_text_embeds,
                          add_time_ids, image_embeds, text_embeds_cloth, guidance_scale, do_cfg, guidance_rescale)

    def _prepare(self, latents, mask, masked_image_latents, pose_latents, cloth_latents, prompt_embeds, add_text_embeds,
                 add_time_ids, image_embeds, text_embeds_cloth, guidance_scale, do_cfg, guidance_rescale):
        L = self.L
        f16 = torch.float16
        B, _, h, w = latents.shape
        Bt = 2 * B if do_cfg else B
        Bg, _, hg, wg = cloth_latents.shape
        dev = self.device
        # the 13-channel concat of src/tryon_pipeline.py:1777 needs every person-side input at the latents' size (the
        # reference fails in torch.cat otherwise); checked before any buffer is written
        for name, t in (("mask", mask), ("masked_image_latents", masked_image_latents), ("pose_latents", pose_latents)):
            if tuple(t.shape[-2:]) != (h, w):
                raise ValueError(f"{name} has spatial size {tuple(t.shape[-2:])}, the latents {(h, w)}: the try-on UNet "
                                 "input concatenates them along channels")
        check_garment_kv_held(self.tryon, None if self.hoist_garment else "TryOnDenoiser(hoist_garment=False)")
        rescale = bool(do_cfg) and guidance_rescale > 0
        key = (B, Bt, Bg, h, w, hg, wg, bool(do_cfg), rescale, tuple(prompt_embeds.shape), tuple(image_embeds.shape),
               tuple(text_embeds_cloth.shape), garment_kv_format(self.tryon))
        fresh = key != getattr(self, "_key", None)
        self._key = key
        self.B, self.Bt, self.Bg, self.h, self.w = B, Bt, Bg, h, w
        self.hg, self.wg = hg, wg
        self.do_cfg = do_cfg
        self.guidance_scale = float(guidance_scale)
        self.rescale = rescale
        self.guidance_rescale = float(guidance_rescale) if rescale else 0.0     # phi applies under CFG only
        if fresh:
            # (re)allocate every static buffer the step graph points at; same-shaped requests reuse them (and the
            # captured graph) and only overwrite their contents
            self.gkv_all = None
            self.latents = torch.empty((B, 4, h, w), dtype=f16, device=dev)
            self.latents_next = torch.empty_like(self.latents)
            self.noise = torch.zeros_like(self.latents)
            self.x_t = torch.zeros((Bt, h, w, CIN_PAD), dtype=f16, device=dev)
            self.x_g = torch.zeros((Bg, hg, wg, CIN_PAD), dtype=f16, device=dev)   # the garment at its own size
            self.t_t = self.t_g = torch.zeros(1, dtype=torch.float32, device=dev)  # one timestep for both UNets
            self.coef = torch.zeros(8, dtype=torch.float32, device=dev)
            self.scale = torch.ones(1, dtype=torch.float32, device=dev)        # Euler's scale_model_input
            self.x0_prev = None                                                # DPM-Solver++ state
            self.step_base = torch.zeros(1, dtype=torch.int32, device=dev)   # step index * Bg (hoisted garment K/V)
            self.ctx_t = self.ctx_g = self.aug = None
            self._graph = self._graph_sig = self.eps = None    # the old graph's memory goes before the K/V budget is read
        self.latents.copy_(latents.to(dev, f16))
        L.nchw_to_nhwc(mask.to(dev, f16).contiguous(), self.x_t, c_off=4)
        L.nchw_to_nhwc(masked_image_latents.to(dev, f16).contiguous(), self.x_t, c_off=5)
        L.nchw_to_nhwc(pose_latents.to(dev, f16).contiguous(), self.x_t, c_off=9)
        L.nchw_to_nhwc(cloth_latents.to(dev, f16).contiguous(), self.x_g, c_off=0)
        self.ctx_t = self.tryon.encode_context(prompt_embeds.to(dev, f16), image_embeds.to(dev, f16), out=self.ctx_t)
        self.ctx_g = self.garment.encode_context(text_embeds_cloth.to(dev, f16), out=self.ctx_g)
        self.aug = self.tryon.aug_embedding(add_text_embeds.to(dev, f16), add_time_ids.to(dev), out=self.aug)

    def set_step_tables(self, scheduler, timesteps, garment_keys=None, cache=None, eta=0.0):
        """Uploads the run's step_plan (timesteps and the step kernel's coefficients, DDIM with `eta`), then runs the
        hoisted garment passes. garment_keys (one hashable per garment of this batch) + cache (GarmentKVCache): garments
        whose K/V of all steps are cached are copied in instead of recomputed — valid only when the caller guarantees that a
        key identifies (cloth latents, text_embeds_cloth); the timestep list and the garment's latent size are added to
        the key here (the person's size does not enter the garment K/V)."""
        plan = step_plan(scheduler, timesteps, self.guidance_scale, self.guidance_rescale, eta)
        vars(self).update(plan.to(self.device)._asdict())                  # kind, coef_table, ..., T
        if self.kind == "dpmpp":
            if self.x0_prev is None:
                self.x0_prev = torch.zeros_like(self.latents)
            self.x0_prev.zero_()
        T = self.T
        self.window = T
        if self.hoist_garment:
            budget = self.max_kv_bytes
            if budget is None:
                # memory this process could still use: free on the device + blocks the caching allocator holds but has
                # not handed out + the K/V buffers of the previous request, which are overwritten in place
                free, _ = torch.cuda.mem_get_info(self.device)
                cached = torch.cuda.memory_reserved(self.device) - torch.cuda.memory_allocated(self.device)
                held = sum(p.numel() * p.element_size() for g in self.gkv_all for p in kv_parts(g)) \
                    if self.gkv_all is not None else 0
                budget = int(0.6 * (free + cached + held))
            per_step = self.kv_bytes_per_step()
            if per_step * T > budget:
                w = max(1, budget // per_step)
                self.window = max(self.garment_chunk, w // self.garment_chunk * self.garment_chunk) if w >= self.garment_chunk else w
        self.base_table = (torch.arange(T, dtype=torch.int32, device=self.device) % self.window) * self.Bg
        if self.hoist_garment:
            use_cache = cache is not None and garment_keys is not None and len(garment_keys) == self.Bg and self.window == T
            if use_cache:
                sig = (tuple(float(t) for t in timesteps), self.hg, self.wg, garment_kv_format(self.tryon))
                full = [(k, sig) for k in garment_keys]
                hit = [cache.get(k) for k in full]
                if all(e is not None for e in hit):
                    if self.gkv_all is None or kv_parts(self.gkv_all[0])[0].shape[0] != T * self.Bg:
                        # first request of this shape (prepare() dropped the static buffers): allocate them from the cached
                        # entries' geometry instead of re-running the garment passes; the step graph is captured afterwards
                        self.gkv_all = [kv_map(src, lambda t: torch.empty((T * self.Bg, *t.shape[1:]), dtype=t.dtype,
                                                                          device=self.device)) for src in hit[0]]
                    for g, e in enumerate(hit):                         # timestep-major rows: row = t * Bg + g
                        for dst, src in zip(self.gkv_all, e):
                            for d, s_ in zip(kv_parts(dst), kv_parts(src)):
                                d.view(T, self.Bg, *d.shape[1:])[:, g].copy_(s_)
                    self.win_start = 0
                    return
            self.precompute_garment(0)
            if use_cache:
                for g, k in enumerate(full):
                    if k not in cache.entries:
                        cache.put(k, [kv_map(kv, lambda t: t.view(T, self.Bg, *t.shape[1:])[:, g].clone())
                                      for kv in self.gkv_all])

    @property
    def garment_chunk(self):
        """Timesteps batched into one hoisted garment-UNet pass (fewer, larger launches); default = up to 64 samples
        per pass."""
        if self._garment_chunk:
            return self._garment_chunk
        return default_garment_chunk(getattr(self, "Bg", 1))

    def kv_bytes_per_step(self):
        """Bytes of garment K/V one denoise step keeps resident: sum over the try-on blocks of Bg * Ng * 2C fp16 (or the
        FP8 format's bytes, garment_kv_bytes_per_step), Ng = the garment's tokens at the block's level (from the cloth
        latents' size)."""
        return self.Bg * garment_kv_bytes_per_step(self.tryon, self.hg, self.wg)

    def precompute_garment(self, win_start=0):
        """The garment-UNet passes of the steps [win_start, win_start + window) of the request (one per timestep), batched,
        then the garment K/V projection of every try-on block for those timesteps: gkv_all[i] = [window*Bg, Ng, 2C] in
        timestep-major order (window = all steps unless the K/V budget forces several windows)."""
        with nvtx_range(f"b200vton.garment_passes[{win_start}:{win_start + self.window}]"):
            self._precompute_garment(win_start)

    def _precompute_garment(self, win_start):
        T_all, Bg = self.T, self.Bg
        T = min(self.window, T_all - win_start)
        rows = min(self.window, T_all) * Bg
        gkv = self.gkv_all            # buffers of an earlier same-shaped request are overwritten in place
        if gkv is not None and kv_parts(gkv[0])[0].shape[0] != rows:
            gkv = None
        self.gkv_all = None
        if gkv is None:
            gkv = [new_garment_kv(self.tryon, rows, ng, b)
                   for b, ng in zip(self.tryon.blocks(), garment_tokens(self.tryon, self.hg, self.wg))]
        hoisted_garment_kv(self.tryon, self.garment, self.x_g, self.ctx_g, self.t_table, win_start, win_start + T,
                           self.garment_chunk, [kv_map(g, lambda t: t[:T * Bg]) for g in gkv])
        self.gkv_all = gkv
        self.win_start = win_start

    def _gkv_pre(self):
        """Hoisted: each try-on block reads the Bg rows from step_base on of its resident garment K/V."""
        return None if self.gkv_all is None else (self.gkv_all, self.Bg, self.step_base)

    def step(self, i, noise=None, use_graph=True):
        """Runs denoise step i (tables from set_step_tables). noise: [B,4,h,w] fp16 variance noise or None."""
        if self.hoist_garment and self.gkv_all is not None and (i // self.window) * self.window != self.win_start:
            self.precompute_garment((i // self.window) * self.window)      # next K/V window (budgeted hoisting)
        return self._run(use_graph, "b200vton.denoise_step", i, noise)

    def _upload(self, i, noise):
        self.t_t.copy_(self.t_table[i:i + 1])
        self.coef.copy_(self.coef_table[i])
        self.step_base.copy_(self.base_table[i:i + 1])
        if self.scale_table is not None:
            self.scale.copy_(self.scale_table[i:i + 1])
        if noise is not None:
            self.noise.copy_(noise)
        else:
            self.noise.zero_()


class SlotDenoiser(_CapturedStep):
    """The denoise step of continuous batching: S slots, each holding one request at its own step index.

    Every buffer is indexed by slot: [S, ...] for persons and garments, [2S, ...] for the try-on batch under CFG (uncond
    row s, cond row S + s). One step is one CUDA graph per capacity: the latent scatter, the garment UNet at batch S with
    per-slot timesteps, the try-on UNet at batch 2S with the garment features of slot s streamed into rows s / S + s, and
    the step kernel that reads one coefficient row per slot (b200vton_cfg_*_step_rows). Before each replay the host
    gathers each slot's timestep / coefficient / input-scale row from the per-step tables into the static buffers, with
    copies issued outside the graph (with B200VTON_PDL_GRAPH every kernel node of the graph is a library kernel).

    Two modes:
      * pages=None (default): the garment UNet runs inside the step at batch S with per-slot timesteps, and the garment
        features of slot s are streamed into try-on rows s / S + s. Nothing is hoisted.
      * pages=P (pool mode, P >= S): the hoisted garment K/V of whole garments live in a pool of P pages, one tensor
        [P*T, Ng, 2C] per try-on block (a GarmentKV8 of P*T rows in the "fp8" garment K/V format) (page p = rows p*T .. p*T + T - 1, so one TMA map per block covers every page and
        the captured graph stays valid while pages are refilled). fill_page runs the T garment passes of one garment
        alone (Bg = 1, TryOnDenoiser's default chunking, hoisted_garment_kv), so a page's bits depend only on the garment
        and the timesteps. The step is the try-on UNet only: slot s reads row page(s)*T + step(s) of the pool through
        b200vton_attention_rows, and an idle slot reads row -1, the zero-K/V closed form (no K/V traffic, and no
        unwritten memory is ever read). The caller (ContinuousTryOnServer) decides which garment is in which page.
      * pages=P, host_pages=Q (pool mode with a host tier): Q more pages in page-locked host memory (HostGarmentKV),
        and 2S more rows at the end of every block's pool tensor, a ring of two rows per slot from R = P*T_page on.
        write_through(p, q) copies a filled device page to host page q on a side stream; a refill of device page p
        waits for that copy on the device. A slot admitted with host_page=q streams: at step i it reads ring row
        R + 2s + (i & 1). Its first row is copied at admission, before the next replay. After each replay the side
        stream copies the next row of every streaming slot into its other ring row, once the step that last read that
        row (the previous replay) is done, and the next replay waits for those copies. Only CUDA events order the two
        streams; the row table is data, so the captured step is the same graph.

    Sampling presets (configure_presets): the slots may follow different StepPlans (scheduler, step count, strength,
    guidance scale, DDPM guidance rescale). Their rows share one table with a kind code per row, a slot names (plan,
    step), and the step is the mixed-kind kernel after the scaled scatter; a slot's result is the bits the per-kind
    kernels give it. In pool mode a page holds T_max rows and a plan of T steps uses its first T.

    Idle slots hold zeros and the identity coefficient row (identity_step_row); their outputs are ignored. No row of one
    slot enters another slot's result, so at a fixed S a request's result does not depend on which slot it runs in or on
    what the other slots hold."""

    ROWS = True
    rescale = False              # refused by configure (the rescale kernel reads one row); per row in configure_presets

    def __init__(self, tryon: UNetEngine, garment: UNetEngine, slots, pages=None, host_pages=None):
        self.tryon, self.garment = tryon, garment
        self.L = tryon.L
        self.device = tryon.device
        self.S = int(slots)
        self.P = None if pages is None else int(pages)
        if self.P is not None and self.P < self.S:
            raise ValueError(f"pool mode needs at least one garment K/V page per slot: {self.P} pages for {self.S} slots")
        self.Q = None if host_pages is None else int(host_pages)
        if self.Q is not None and (self.P is None or self.Q < 1):
            raise ValueError(f"a host tier of {self.Q} garment K/V pages needs pool mode (pages=P) and at least one page")
        self.garment_chunk = default_garment_chunk(1)
        self.page = [None] * self.S                 # pool mode: the page each slot's request reads
        self.host_page = [None] * self.S            # host tier: the host page a streaming slot reads
        self.host = None
        self.pool = None
        self._side = None                           # host tier: the copy stream and its events (made at first use)
        self._page_rows = {}                        # device page -> rows its last fill wrote
        self._page_copied = {}                      # device page -> event of its last write-through
        self._host_written = {}                     # host page -> event of its last write-through
        self._streamed = [0, 0]                     # rows and bytes copied into the ring since take_streamed()
        self._key = None
        self.ctx_t = None
        self.plans = self.kind_table = None         # configure_presets: the plans and the kind of every table row

    def _needs(self, kind):
        names = ["b200vton_cfg_step_mixed_rows" if kind == "mixed" else
                 "b200vton_cfg_ddpm_step_rows" if kind == "ddpm" else "b200vton_cfg_solver_step_rows"]
        if kind in ("euler", "mixed"):
            names.append("b200vton_nchw_to_nhwc_scaled_rows")
        if self.P is not None:
            names.append("b200vton_attention_rows")
        return names

    def _check_kv_format(self):
        check_garment_kv_held(self.tryon, "continuous batching without a garment K/V pool (pages=None)"
                              if self.P is None else None)

    def configure(self, scheduler, timesteps, h, w, guidance_scale=2.0, do_cfg=True, eta=0.0, guidance_rescale=0.0):
        """Per-step tables of the run (one scheduler, one step count for every request) and the static buffers of a
        person latent size h x w (the garment has the same size). Raises before any launch when the library lacks a
        per-slot kernel the scheduler needs, and for guidance_rescale > 0 (its per-sample statistics are fused with the
        single-row DDPM kernel only)."""
        if guidance_rescale and guidance_rescale > 0:
            raise NotImplementedError("guidance_rescale > 0 is not supported by continuous batching: the rescale kernel "
                                      "reads one coefficient row for the whole batch")
        plan = step_plan(scheduler, timesteps, guidance_scale, eta=eta)    # row T: idle slots
        self._check_kv_format()
        for name in self._needs(plan.kind):
            if not self.L.has_symbol(name):
                raise NotImplementedError(f"continuous batching needs {name}, which this library binding does not export")
        vars(self).update(plan.to(self.device)._asdict())                  # kind, coef_table, ..., T
        self.plans = self.kind_table = None
        self.T_page = self.T
        self._allocate(h, w, do_cfg)
        self.gather([None] * self.S)

    def configure_presets(self, plans, h, w, do_cfg=True):
        """Per-step tables of several runs at once (sampling presets), stepped together by the mixed-kind step kernel
        (b200vton_cfg_step_mixed_rows): plans is a list of StepPlan (step_plan, DDPM rows may carry a guidance
        rescale). Their rows are concatenated into one coefficient / timestep / input-scale table (scale 1 for the
        kinds that do not scale their input, which the scaled scatter applies exactly) with one kind code per row
        (MIXED_KIND_CODES) and one identity row at the end for idle slots; plan j's step i is row base[j] + i. In pool
        mode a page holds T_max = the largest T of the plans rows. Raises before any launch when the library lacks an
        entry point this needs."""
        plans = list(plans)
        if not plans:
            raise ValueError("configure_presets needs at least one StepPlan")
        for name in self._needs("mixed"):
            if not self.L.has_symbol(name):
                raise NotImplementedError(f"sampling presets need {name}, which this library binding does not export")
        self._check_kv_format()
        f32 = torch.float32
        idle = plans[0].kind
        self.base, n = [], 0
        for p in plans:
            self.base.append(n)
            n += p.T
        self.idle = n
        coef = torch.cat([p.coef_table[:p.T].cpu() for p in plans] + [torch.tensor([identity_step_row(idle)], dtype=f32)])
        t = torch.cat([p.t_table[:p.T].cpu() for p in plans] + [torch.zeros(1, dtype=f32)])
        scale = torch.cat([torch.ones(p.T, dtype=f32) if p.scale_table is None else p.scale_table[:p.T].cpu()
                           for p in plans] + [torch.ones(1, dtype=f32)])
        kinds = [MIXED_KIND_CODES[p.kind] for p in plans for _ in range(p.T)] + [MIXED_KIND_CODES[idle]]
        dev = self.device
        self.coef_table, self.t_table, self.scale_table = coef.to(dev), t.to(dev), scale.to(dev)
        self.kind_table = torch.tensor(kinds, dtype=torch.int32).to(dev)
        self.plans = plans
        self.kind, self.T, self.step_draws, self.noise_applied = "mixed", None, None, None
        self.T_page = max(p.T for p in plans)
        self._allocate(h, w, do_cfg)
        self.gather([None] * self.S)

    def _allocate(self, h, w, do_cfg):
        """The static buffers of a person latent size h x w (the garment has the same size), kept while the key holds."""
        dev, f16, f32 = self.device, torch.float16, torch.float32
        self.do_cfg, self.h, self.w = bool(do_cfg), h, w
        S = self.S
        self.Bt = 2 * S if do_cfg else S
        key = (S, h, w, self.do_cfg, self.kind) + (() if self.P is None else (self.P, self.T_page,
                                                                               garment_kv_format(self.tryon)))
        if key != self._key:
            self.ctx_t = self.ctx_g = self.aug = None
            self.latents = torch.zeros((S, 4, h, w), dtype=f16, device=dev)
            self.latents_next = torch.zeros_like(self.latents)
            self.noise = torch.zeros_like(self.latents)
            self.x0_prev = torch.zeros_like(self.latents) if self.kind in ("dpmpp", "mixed") else None
            self.x_t = torch.zeros((self.Bt, h, w, CIN_PAD), dtype=f16, device=dev)
            if self.P is None:
                self.x_g = torch.zeros((S, h, w, CIN_PAD), dtype=f16, device=dev)
                self.t_g = torch.zeros(S, dtype=f32, device=dev)
            else:
                # allocated once (the old pool is released first); every page is written by fill_page before a slot's
                # row names it
                self.release_host()
                self._page_rows.clear()
                self.x_g = self.t_g = self.pool = None
                if self.Q is not None:         # host first: a failed page-lock raises before the device pool grows
                    self.host = HostGarmentKV(self.tryon, self.Q, self.T_page, h, w)
                self.ring = self.P * self.T_page
                ring_rows = 0 if self.Q is None else 2 * S
                self.pool = [new_garment_kv(self.tryon, self.ring + ring_rows, ng, b)
                             for b, ng in zip(self.tryon.blocks(), garment_tokens(self.tryon, h, w))]
                self.rows = torch.full((S,), -1, dtype=torch.int32, device=dev)
                self.page = [None] * S
                self.host_page = [None] * S
            self.t_t = torch.zeros(self.Bt, dtype=f32, device=dev)
            self.coef = torch.zeros((S, 8), dtype=f32, device=dev)
            self.scale = torch.ones(S, dtype=f32, device=dev)
            self.kinds = torch.zeros(S, dtype=torch.int32, device=dev) if self.kind == "mixed" else None
            self._key = key                    # last: a failed allocation leaves the key to be allocated again

    def gather(self, steps):
        """steps: per slot, the step index of its request or None (idle); after configure_presets, (plan index, step
        index) or None. Copies the slot's row of the tables (the idle row when idle) into the graph's static t / coef /
        scale / kind buffers (t at rows s and S + s of the try-on batch)."""
        if self.plans is None:
            step_of = list(steps)
            rows = [self.T if i is None else int(i) for i in steps]
        else:
            step_of, rows = [], []
            for s, e in enumerate(steps):
                if e is not None and not (0 <= e[0] < len(self.plans) and 0 <= e[1] < self.plans[e[0]].T):
                    raise ValueError(f"slot {s}: (plan, step) {tuple(e)} outside the configured plans")
                step_of.append(None if e is None else int(e[1]))
                rows.append(self.idle if e is None else self.base[e[0]] + int(e[1]))
        idx = torch.tensor(rows, dtype=torch.long).to(self.device)
        torch.index_select(self.coef_table, 0, idx, out=self.coef)
        t = self.t_table.index_select(0, idx)
        if self.t_g is not None:
            self.t_g.copy_(t)
        self.t_t.copy_(t.repeat(self.Bt // self.S))
        if self.scale_table is not None:
            torch.index_select(self.scale_table, 0, idx, out=self.scale)
        if self.kind_table is not None:
            torch.index_select(self.kind_table, 0, idx, out=self.kinds)
        if self.P is not None:
            self.rows.copy_(torch.tensor(self.kv_rows(step_of), dtype=torch.int32))

    def kv_rows(self, step_of):
        """Pool mode: the pool row of every slot at its step index (None: idle). Slot s reads row page(s) * T_page +
        step(s); streaming from the host tier, ring row P * T_page + 2s + (step & 1); idle, row -1 (zero K/V)."""
        rows, streaming = [], []
        for s, i in enumerate(step_of):
            if i is None:
                rows.append(-1)
            elif self.host_page[s] is not None:
                rows.append(self.ring + 2 * s + (int(i) & 1))
                streaming.append(s)
            elif self.page[s] is None:
                raise ValueError(f"slot {s} is at step {i} but holds no garment K/V page")
            else:
                rows.append(self.page[s] * self.T_page + int(i))
        if any(not -1 <= r < self.ring for s, r in enumerate(rows) if s not in streaming):   # the device pages' rows
            raise ValueError(f"garment K/V rows {rows} outside [-1, {self.ring})")
        return rows

    def fill_page(self, p, cloth_latents, text_embeds_cloth, t_table=None):
        """Pool mode: writes the garment K/V of all T steps of one garment (cloth_latents [1,4,h,w], text_embeds_cloth
        [1,77,X]) into page p: its T garment-UNet passes at Bg = 1, chunked as TryOnDenoiser chunks them, so the page
        holds the bits TryOnDenoiser's gkv_all holds for that garment alone. Runs eagerly (not in the step graph).
        t_table: after configure_presets, the timesteps of the plan the page is filled for (its first rows then hold
        them; required), else the configured run's."""
        if self.P is None or self.pool is None:
            raise RuntimeError("SlotDenoiser.fill_page needs pool mode (pages=P) and configure() first")
        if not 0 <= p < self.P:
            raise ValueError(f"page {p} outside [0, {self.P})")
        if t_table is None:
            if self.plans is not None:
                raise ValueError("fill_page after configure_presets needs the timesteps of the page's plan")
            t_table, T = self.t_table, self.T
        else:
            t_table = t_table.to(self.device, torch.float32)
            T = t_table.shape[0]
            if not 0 < T <= self.T_page:
                raise ValueError(f"{T} timesteps do not fit a page of {self.T_page} rows")
        if tuple(cloth_latents.shape[-2:]) != (self.h, self.w):
            raise ValueError(f"cloth_latents has spatial size {tuple(cloth_latents.shape[-2:])}, the server's latents "
                             f"{(self.h, self.w)}")
        dev, f16, Tp = self.device, torch.float16, self.T_page
        copied = self._page_copied.pop(p, None)
        if copied is not None:                  # the page's write-through reads it: the refill waits on the device
            torch.cuda.current_stream(dev).wait_event(copied)
        self._page_rows[p] = T
        with nvtx_range(f"b200vton.garment_page_fill[{p}]"):
            x_g = torch.zeros((1, self.h, self.w, CIN_PAD), dtype=f16, device=dev)
            self.L.nchw_to_nhwc(cloth_latents[:1].to(dev, f16).contiguous(), x_g, c_off=0)
            ctx_g = self.garment.encode_context(text_embeds_cloth[:1].to(dev, f16))
            hoisted_garment_kv(self.tryon, self.garment, x_g, ctx_g, t_table, 0, T, self.garment_chunk,
                               [kv_map(g, lambda t: t[p * Tp:p * Tp + T]) for g in self.pool])

    def _rows(self, s):
        return (s, self.S + s) if self.do_cfg else (s,)

    def admit(self, s, latents, mask, masked_image_latents, pose_latents, cloth_latents, prompt_embeds, add_text_embeds,
              add_time_ids, image_embeds, text_embeds_cloth, page=None, host_page=None):
        """Writes one request into slot s, and only its rows. latents [1,4,h,w]; mask [1,1,h,w]; masked_image_latents,
        pose_latents, cloth_latents [1,4,h,w]; prompt_embeds [n,77,X], add_text_embeds [n,P], add_time_ids [n,6],
        image_embeds [n,16,X] with n = 2 ([uncond ; cond]) under CFG, else 1 (mask, masked_image_latents and
        pose_latents may have n rows too); text_embeds_cloth [1,77,X]. Pool mode: `page` is the filled page of the
        request's garment (cloth_latents and text_embeds_cloth are then not read); with a host tier, `host_page`
        instead is the host page the slot streams from, from step 0 on (its first row is copied here)."""
        L, dev, f16 = self.L, self.device, torch.float16
        if host_page is not None:
            if self.host is None or page is not None or not 0 <= host_page < self.Q:
                raise ValueError(f"admit streams from a host page in [0, {self.Q}) of a host tier, instead of a device "
                                 f"page: got host_page={host_page}, page={page}")
        elif self.P is not None and (page is None or not 0 <= page < self.P):
            raise ValueError(f"pool mode: admit needs the page of the request's garment in [0, {self.P}), got {page}")
        for name, t in (("latents", latents), ("mask", mask), ("masked_image_latents", masked_image_latents),
                        ("pose_latents", pose_latents), ("cloth_latents", cloth_latents)):
            if tuple(t.shape[-2:]) != (self.h, self.w):
                raise ValueError(f"{name} has spatial size {tuple(t.shape[-2:])}, the server's latents {(self.h, self.w)}")
        rows = self._rows(s)
        if self.ctx_t is None:
            ni = image_embeds.shape[1] if self.tryon.ip_tokens else 0
            self.ctx_t = [(torch.zeros((self.Bt, prompt_embeds.shape[1], 2 * b.c), dtype=f16, device=dev),
                           torch.zeros((self.Bt, ni, 2 * b.c), dtype=f16, device=dev) if ni else None)
                          for b in self.tryon.blocks()]
            if self.P is None:
                self.ctx_g = [(torch.zeros((self.S, text_embeds_cloth.shape[1], 2 * b.c), dtype=f16, device=dev), None)
                              for b in self.garment.blocks()]
            self.aug =torch.zeros((self.Bt, self.tryon.ae[2].shape[0]), dtype=f16, device=dev)
        self.latents[s].copy_(latents[0].to(dev, f16))
        for j, r in enumerate(rows):
            x = self.x_t[r:r + 1]
            for t, c_off in ((mask, 4), (masked_image_latents, 5), (pose_latents, 9)):
                row = t[j:j + 1] if t.shape[0] == len(rows) else t[:1]
                L.nchw_to_nhwc(row.to(dev, f16).contiguous(), x, c_off=c_off)
            self.tryon.encode_context(prompt_embeds[j:j + 1].to(dev, f16), image_embeds[j:j + 1].to(dev, f16),
                                      out=[(kt[r:r + 1], None if ki is None else ki[r:r + 1]) for kt, ki in self.ctx_t])
            self.tryon.aug_embedding(add_text_embeds[j:j + 1].to(dev, f16), add_time_ids[j:j + 1].to(dev),
                                     out=self.aug[r:r + 1])
        if self.P is None:
            L.nchw_to_nhwc(cloth_latents[:1].to(dev, f16).contiguous(), self.x_g[s:s + 1], c_off=0)
            self.garment.encode_context(text_embeds_cloth[:1].to(dev, f16),
                                        out=[(kv[s:s + 1], None) for kv, _ in self.ctx_g])
        elif host_page is not None:
            self.page[s], self.host_page[s] = None, int(host_page)
            self._stream_rows([(s, 0)], after_last_step=True)
        else:
            self.page[s] = int(page)
        if self.x0_prev is not None:
            self.x0_prev[s].zero_()

    def release(self, s):
        """Frees slot s: its latents, state and input channels go back to zeros (the context rows keep finite values
        that no other slot reads); in pool mode it no longer names a page."""
        for buf in (self.latents, self.latents_next, self.noise, self.x0_prev, self.x_g):
            if buf is not None:
                buf[s].zero_()
        for r in self._rows(s):
            self.x_t[r].zero_()
        self.page[s] = None
        self.host_page[s] = None

    # ---- host tier --------------------------------------------------------------------------------
    def _copy_streams(self):
        """The host tier's side streams and the events that order them against the step: "ring" copies rows into the
        ring (host to device), "write" copies filled pages to the host (device to host), so that a page's write-through
        never holds up the next step's rows; "replayed": the last two replays' events (by replay parity); "ring_ready":
        the ring copies the next replay waits for."""
        if self._side is None:
            ev = torch.cuda.Event
            self._side = dict(ring=torch.cuda.Stream(device=self.device), write=torch.cuda.Stream(device=self.device),
                              replayed=[ev(), ev()], n=0, ring_ready=ev(), ring_pending=False)
        return self._side

    def _stream_rows(self, loads, after_last_step):
        """Copies host row q*T_page + i of each (slot, step i) in `loads` into ring row R + 2s + (i & 1) on the ring
        stream, and makes the next replay wait for them. The ring stream first waits for the step that last read those
        ring rows: the latest replay when a slot is admitted (after_last_step), else the one before it (the copies of
        step i + 1 then run beside step i), and for a write-through into the host page still in flight."""
        side = self._copy_streams()
        stream = side["ring"]
        k = side["n"] - (1 if after_last_step else 2)         # the replay to wait for (side["n"] replays so far)
        if k >= 0:
            stream.wait_event(side["replayed"][k & 1])
        with torch.cuda.stream(stream):
            for s, i in loads:
                q = self.host_page[s]
                written = self._host_written.get(q)
                if written is not None:
                    stream.wait_event(written)
                src, dst = q * self.T_page + i, self.ring + 2 * s + (i & 1)
                for pool_kv, host_kv in zip(self.pool, self.host.blocks):
                    self._streamed[1] += copy_kv_rows(pool_kv, dst, host_kv, src)
                self._streamed[0] += 1
            side["ring_ready"].record(stream)
        side["ring_pending"] = True

    def write_through(self, p, q):
        """Copies device page p (the rows of its last fill) to host page q on the write stream, after the work the
        current stream has enqueued (the fill) and after the ring copies issued so far (which may read host page q's
        previous garment). Until that copy is done, a refill of page p waits for it on the device, and rows streamed
        from host page q wait for it on the ring stream. The host does not wait."""
        if self.host is None or not (0 <= p < self.P and 0 <= q < self.Q) or p not in self._page_rows:
            raise ValueError(f"write_through needs a host tier, a filled device page in [0, {self.P}) and a host page "
                             f"in [0, {self.Q}): got {p}, {q}")
        side = self._copy_streams()
        stream = side["write"]
        filled = torch.cuda.Event()
        filled.record(torch.cuda.current_stream(self.device))
        stream.wait_event(filled)
        stream.wait_stream(side["ring"])
        T, Tp = self._page_rows[p], self.T_page
        with torch.cuda.stream(stream):
            for host_kv, pool_kv in zip(self.host.blocks, self.pool):
                copy_kv_rows(host_kv, q * Tp, pool_kv, p * Tp, T)
            done = torch.cuda.Event()
            done.record(stream)
        self._page_copied[p] = self._host_written[q] = done

    def take_streamed(self):
        """(rows, bytes) copied from the host tier into the ring since the last call."""
        out, self._streamed = tuple(self._streamed), [0, 0]
        return out

    def release_host(self):
        """Waits for the side streams' copies, then unregisters and drops the host tier's memory."""
        if self._side is not None:
            self._side["ring"].synchronize()
            self._side["write"].synchronize()
        self._page_copied.clear()
        self._host_written.clear()
        if self.host is not None:
            self.host.release()
            self.host = None

    def _gkv_pre(self):
        return None if self.P is None else (self.pool, self.rows)

    def step(self, steps, noises=None, use_graph=True):
        """One denoise step of every occupied slot. steps: per slot, its request's step index or None (idle); noises:
        {slot: [1,4,h,w] variance noise} for the slots whose scheduler step applies one. Returns the latents [S,4,h,w].
        With a host tier, the next row of every streaming slot is then copied into its ring beside the next step."""
        if self.ctx_t is None:
            raise RuntimeError("SlotDenoiser.step before any admission")
        out = self._run(use_graph, "b200vton.slot_denoise_step", steps, noises)
        if self.host is not None and self._side is not None:
            side = self._side
            side["replayed"][side["n"] & 1].record(torch.cuda.current_stream(self.device))
            side["n"] += 1
            loads = []
            for s, e in enumerate(steps):
                if e is None or self.host_page[s] is None:
                    continue
                i = int(e) if self.plans is None else int(e[1])
                T = self.T if self.plans is None else self.plans[e[0]].T
                if i + 1 < T:
                    loads.append((s, i + 1))
            if loads:
                self._stream_rows(loads, after_last_step=False)
        return out

    def _upload(self, steps, noises):
        if self._side is not None and self._side["ring_pending"]:     # the ring rows this step reads
            torch.cuda.current_stream(self.device).wait_event(self._side["ring_ready"])
            self._side["ring_pending"] = False
        self.gather(steps)
        self.noise.zero_()
        for s, n in (noises or {}).items():
            self.noise[s].copy_(n[0])
