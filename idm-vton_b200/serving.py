"""Request front-end for the try-on engine (SURVEY.md 8f item 4): replaces the reference's DataLoader loop
(inference.py:309-341, 337-419: fixed batches in dataset order, the garment UNet re-run for every sample of every batch)
with batching BY GARMENT and reuse of garment work across requests.

  * requests that wear the same garment are batched together: the garment UNet then runs at batch 1 and its K/V of every
    denoise step are indexed by all persons of the batch (BASELINE config 3);
  * each garment is VAE-encoded ONCE (one posterior sample per garment instead of one per call) and the hoisted garment
    K/V of all denoise steps are kept in an LRU cache (denoise.GarmentKVCache), so a garment seen before costs a few
    device-to-device copies instead of `num_inference_steps` garment-UNet passes.
Everything per person (noise, masks, pose, prompts) is exactly what `StableDiffusionXLInpaintPipeline.__call__` does; the
only semantic difference from calling the pipeline per DataLoader batch is the once-per-garment posterior sample, which is
why the cache is a property of this front-end and not of the pipeline (off unless a server installs it).
Single-threaded by design, like the reference pipeline (one CUDA stream, one denoiser / graph per process).
"""
import collections
import dataclasses
from typing import Any, Hashable, Optional

import torch

from .denoise import GarmentKVCache


@dataclasses.dataclass
class TryOnRequest:
    """One person x one garment. Tensors follow the keyword set of inference.py:397-414 for a batch of 1."""
    garment_id: Hashable
    image: torch.Tensor                 # [3,H,W] in [0,1]
    mask_image: torch.Tensor            # [1,H,W]
    pose_img: torch.Tensor              # [3,H,W] in [-1,1]
    prompt_embeds: torch.Tensor         # [77,2048]
    negative_prompt_embeds: torch.Tensor
    pooled_prompt_embeds: torch.Tensor  # [1280]
    negative_pooled_prompt_embeds: torch.Tensor
    # garment side (needed the first time a garment_id is seen; ignored afterwards)
    cloth: Optional[torch.Tensor] = None             # [3,H,W] in [-1,1]
    ip_adapter_image: Optional[torch.Tensor] = None  # [3,224,224] CLIP-preprocessed garment image
    text_embeds_cloth: Optional[torch.Tensor] = None  # [77,2048]
    ticket: Any = None
    seed: Optional[int] = None          # ContinuousTryOnServer: this request's generator (TryOnServer ignores it)


def _encode_garment(pipe, src, seed, device, dtype):
    """ONE posterior sample per garment, from a generator of its own (seeded with the server's seed): the per-request
    generator must see the same stream whether or not the garment was already known."""
    cloth = src.cloth[None].to(device=device, dtype=dtype)
    gen = torch.Generator(device).manual_seed(seed) if seed is not None else None
    latents = pipe._encode_vae_image(cloth, generator=gen)
    return dict(latents=latents, ip_adapter_image=src.ip_adapter_image[None].to(device),
                text_embeds_cloth=src.text_embeds_cloth[None].to(device=device, dtype=dtype))


def _seeded_global_rng(device, seed):
    """The reference draws the pose latents' posterior sample from the GLOBAL generator (src/tryon_pipeline.py:1646
    passes no generator): with a seed, the global CPU / device generators are forked around the draw and seeded (their
    state outside is untouched); without one, the global generators are used as they are."""
    import contextlib
    if seed is None:
        return contextlib.nullcontext()
    dev_idx = [torch.device(device).index or 0] if torch.device(device).type == "cuda" else []

    @contextlib.contextmanager
    def ctx():
        with torch.random.fork_rng(devices=dev_idx):
            torch.manual_seed(seed)
            yield
    return ctx()


class TryOnServer:
    def __init__(self, pipe, height=1024, width=768, num_inference_steps=30, guidance_scale=2.0, max_batch=8, seed=None,
                 garment_cache_bytes=40 << 30, output_type="pt"):
        self.pipe = pipe
        self.height, self.width = height, width
        self.num_inference_steps, self.guidance_scale = num_inference_steps, guidance_scale
        self.max_batch = max_batch
        self.seed = seed
        self.output_type = output_type
        self.queue = collections.OrderedDict()      # garment_id -> deque of requests (arrival order inside a garment)
        self.garments = {}                          # garment_id -> dict(latents, ip_adapter_image, text_embeds_cloth)
        self._next_ticket = 0
        self.stats = collections.Counter()
        if garment_cache_bytes:
            pipe.garment_cache = GarmentKVCache(garment_cache_bytes)

    # ---------------------------------------------------------------------------------------------
    def submit(self, req: TryOnRequest):
        if req.garment_id not in self.garments and req.garment_id not in self.queue and \
                (req.cloth is None or req.ip_adapter_image is None or req.text_embeds_cloth is None):
            raise ValueError(f"garment {req.garment_id!r} is new: cloth, ip_adapter_image and text_embeds_cloth are required")
        req.ticket = self._next_ticket
        self._next_ticket += 1
        self.queue.setdefault(req.garment_id, collections.deque()).append(req)
        return req.ticket

    def pending(self):
        return sum(len(q) for q in self.queue.values())

    def _next_batch(self):
        """Oldest waiting request decides the garment; up to max_batch requests of that garment go together."""
        gid = min(self.queue, key=lambda g: self.queue[g][0].ticket)
        q = self.queue[gid]
        batch = [q.popleft() for _ in range(min(self.max_batch, len(q)))]
        if not q:
            del self.queue[gid]
        return gid, batch

    def _garment(self, gid, batch, device, dtype):
        g = self.garments.get(gid)
        if g is None:
            g = _encode_garment(self.pipe, next(r for r in batch if r.cloth is not None), self.seed, device, dtype)
            self.garments[gid] = g
            self.stats["garments_encoded"] += 1
        return g

    @torch.no_grad()
    def step(self):
        """Runs ONE batch; returns {ticket: image}."""
        if not self.queue:
            return {}
        gid, batch = self._next_batch()
        pipe = self.pipe
        device = pipe._execution_device
        dtype = pipe.unet.dtype
        gen = torch.Generator(device).manual_seed(self.seed) if self.seed is not None else None
        g = self._garment(gid, batch, device, dtype)
        stack = lambda name, dt=None: torch.stack([getattr(r, name) for r in batch]).to(device=device, dtype=dt)  # noqa: E731
        # the pose latents' sample comes from the global generator: seeded around the call (_seeded_global_rng), so a
        # seeded server is reproducible
        with _seeded_global_rng(device, self.seed):
            images = pipe(prompt_embeds=stack("prompt_embeds", dtype), negative_prompt_embeds=stack("negative_prompt_embeds", dtype),
                          pooled_prompt_embeds=stack("pooled_prompt_embeds", dtype),
                          negative_pooled_prompt_embeds=stack("negative_pooled_prompt_embeds", dtype),
                          num_inference_steps=self.num_inference_steps, generator=gen, strength=1.0,
                          pose_img=stack("pose_img", dtype), text_embeds_cloth=g["text_embeds_cloth"], cloth=g["latents"],
                          mask_image=stack("mask_image"), image=stack("image"), height=self.height, width=self.width,
                          ip_adapter_image=g["ip_adapter_image"], guidance_scale=self.guidance_scale,
                          output_type=self.output_type, garment_keys=[gid])[0]
        self.stats["batches"] += 1
        self.stats["images"] += len(batch)
        return {r.ticket: images[i] for i, r in enumerate(batch)}

    def run(self):
        """Drains the queue; returns {ticket: image}."""
        out = {}
        while self.queue:
            out.update(self.step())
        return out


class ContinuousTryOnServer:
    """Continuous batching: requests join and leave the denoise batch at every step (denoise.SlotDenoiser).

    The server has `slots` slots. Each `step()` admits waiting requests into free slots (lowest slot first, in ticket
    order), replays ONE denoise step in which every occupied slot advances its own request by one step, then VAE-decodes
    the requests that finished (one decode for all of them) and frees their slots. A request therefore waits for a free
    slot, not for a whole batch, and a batch that is not full fills up at the next step.

    One scheduler (the pipeline's), one `num_inference_steps` and one guidance scale for every request, and one person
    size (height x width); the garment must have the same latent size. Garments are VAE-encoded once per garment_id
    exactly as TryOnServer does.

    Garment work, two modes:
      * garment_kv_bytes=None (default): the garment UNet runs inside every step at batch `slots` (no hoisting and no
        GarmentKVCache: requests at different phases need the garment K/V of different timesteps).
      * garment_kv_bytes=N (pool mode): a pool of P = N // page_bytes pages of hoisted garment K/V (SlotDenoiser with
        pages=P), page_bytes = T * kv_bytes_per_step of one garment (9.44 GB at 768x1024 with 30 steps, computed from the
        shapes). Admitting a request pins its garment's page; on a miss the garment's T passes fill a free page, or the
        least recently used unpinned one, eagerly at admission before that step's replay. Slots with the same garment
        share its page; a retired request unpins it and the page stays resident, so a later request for that garment
        runs no garment pass at all. The step is then the try-on UNet only. P < slots is refused (ValueError naming the
        page size) before any launch. `stats` counts garment_page_fills and garment_page_hits.

    RNG: each request owns a generator seeded with `req.seed` (the server's seed when None; unseeded when both are None)
    and draws in the order the pipeline draws for a batch of one: the initial noise, the masked image's VAE sample, the
    pose sample from the global generator (forked and seeded with the same seed, as TryOnServer does), then the variance
    noise of every step whose scheduler step draws one. A request's result is then independent of arrival order, slot
    and neighbours (at a fixed number of slots): its final latents always, its image when it finishes at a step of its
    own (requests finishing at the same step share one VAE decode).
    `eta`: DDIM's eta, as the pipeline's `__call__` takes it (0 = deterministic DDIM, 1 = DDPM-like variance).
    Refused: guidance_rescale (not a parameter here), schedulers other than DDPM / DDIM / Euler / DPM-Solver++, and a
    library without the per-slot step kernels or, in pool mode, without b200vton_attention_rows (NotImplementedError
    naming the symbol, before any launch)."""

    def __init__(self, pipe, height=1024, width=768, slots=4, num_inference_steps=30, guidance_scale=2.0, seed=None,
                 output_type="pt", eta=0.0, garment_kv_bytes=None):
        self.pipe = pipe
        self.height, self.width = height, width
        self.S = int(slots)
        self.num_inference_steps, self.guidance_scale = num_inference_steps, guidance_scale
        self.seed = seed
        self.output_type = output_type
        self.eta = float(eta)                        # DDIM's eta (the pipeline's `eta`; other schedulers ignore it)
        self.guidance_rescale = 0.0
        vsf = pipe.vae_scale_factor
        self.latent_size = (height // vsf, width // vsf)
        self.waiting = collections.deque()
        self.slots = [None] * self.S                 # per slot: dict(req, gen, step) or None
        self.garments = {}
        self.den = None
        self.garment_kv_bytes = None if garment_kv_bytes is None else int(garment_kv_bytes)
        self.page_of = collections.OrderedDict()     # pool mode: garment_id -> page, least recently admitted first
        self.pins = collections.Counter()            # pool mode: page -> slots whose request reads it
        self.free_pages = []
        self.last_latents = {}                       # ticket -> final latents of the requests the last step() finished
        self._next_ticket = 0
        self.stats = collections.Counter()

    # ---------------------------------------------------------------------------------------------
    def submit(self, req: TryOnRequest):
        known = req.garment_id in self.garments or any(r.garment_id == req.garment_id for r in self.waiting) or any(
            e is not None and e["req"].garment_id == req.garment_id for e in self.slots)
        if not known:
            if req.cloth is None or req.ip_adapter_image is None or req.text_embeds_cloth is None:
                raise ValueError(f"garment {req.garment_id!r} is new: cloth, ip_adapter_image and text_embeds_cloth are "
                                 "required")
            vsf = self.pipe.vae_scale_factor
            size = (req.cloth.shape[-2] // vsf, req.cloth.shape[-1] // vsf)
            if size != self.latent_size:
                raise ValueError(f"garment {req.garment_id!r} has latent size {size}, the server's persons "
                                 f"{self.latent_size}: every slot runs the garment UNet at one size")
        req.ticket = self._next_ticket
        self._next_ticket += 1
        self.waiting.append(req)
        return req.ticket

    def pending(self):
        return len(self.waiting) + sum(e is not None for e in self.slots)

    # ---------------------------------------------------------------------------------------------
    def _make_denoiser(self, pages=None):
        from .denoise import SlotDenoiser
        return SlotDenoiser(self.pipe.unet.engine(), self.pipe.unet_encoder.engine(), self.S, pages=pages)

    def page_bytes(self, T=None):
        """Pool mode: bytes of one garment's page, the hoisted K/V of all T steps at Bg = 1 (from the shapes)."""
        from .denoise import garment_kv_bytes_per_step
        T = self.num_inference_steps if T is None else T
        return T * garment_kv_bytes_per_step(self.pipe.unet.engine(), *self.latent_size)

    def _pages(self, T):
        """Pool mode: the number of pages the budget holds; refuses fewer than one per slot."""
        page = self.page_bytes(T)
        P = self.garment_kv_bytes // page
        if P < self.S:
            raise ValueError(f"garment_kv_bytes={self.garment_kv_bytes} holds {P} garment K/V pages of {page} bytes "
                             f"({page / 1e9:.2f} GB: {T} steps at latent size {self.latent_size}); pool mode needs at "
                             f"least one page per slot ({self.S}, i.e. {self.S * page} bytes)")
        return P

    def _reset_pages(self, P):
        self.page_of.clear()
        self.pins.clear()
        self.free_pages = list(range(P))

    def _configure(self):
        """Timesteps and per-step tables of the run (the pipeline's own timestep selection at strength 1); checks every
        refusal before the first launch."""
        from .pipeline import retrieve_timesteps
        pipe = self.pipe
        pipe._guidance_scale = self.guidance_scale
        timesteps, n = retrieve_timesteps(pipe.scheduler, self.num_inference_steps, pipe._execution_device)
        timesteps, n = pipe.get_timesteps(n, 1.0, pipe._execution_device)
        self.timesteps = timesteps
        if self.den is None:
            if self.garment_kv_bytes is None:
                self.den = self._make_denoiser()
            else:
                P = self._pages(len(timesteps))
                self.den = self._make_denoiser(pages=P)
                self._reset_pages(P)
        self.den.configure(pipe.scheduler, timesteps, *self.latent_size, guidance_scale=self.guidance_scale,
                           do_cfg=pipe.do_classifier_free_guidance, eta=self.eta, guidance_rescale=self.guidance_rescale)
        self.T = self.den.T
        self._configured = True

    def _garment(self, req, device, dtype):
        g = self.garments.get(req.garment_id)
        if g is None:
            src = req if req.cloth is not None else next(
                r for r in self.waiting if r.garment_id == req.garment_id and r.cloth is not None)
            g = _encode_garment(self.pipe, src, self.seed, device, dtype)
            emb = self.pipe.prepare_ip_adapter_image_embeds(g["ip_adapter_image"], device, 1)
            g["image_embeds"] = self.pipe.unet.encoder_hid_proj(emb).to(dtype)         # Resampler, once per garment
            self.garments[req.garment_id] = g
            self.stats["garments_encoded"] += 1
        return g

    def _prepare_request(self, req, gen):
        """The pipeline's own preparation of one person (batch 1, strength 1): pre-processing, initial latents, mask and
        masked-image latents, pose latents, prompt and added-condition embeddings — drawing from `gen` in the
        pipeline's order. Returns the keyword arguments of SlotDenoiser.admit except the garment's."""
        pipe = self.pipe
        device, dtype = pipe._execution_device, pipe.unet.dtype
        do_cfg = pipe.do_classifier_free_guidance
        H, W = self.height, self.width
        pe, npe, ppe, nppe = pipe.encode_prompt(
            prompt=None, device=device, num_images_per_prompt=1, do_classifier_free_guidance=do_cfg,
            prompt_embeds=req.prompt_embeds[None].to(device=device, dtype=dtype),
            negative_prompt_embeds=req.negative_prompt_embeds[None].to(device=device, dtype=dtype),
            pooled_prompt_embeds=req.pooled_prompt_embeds[None].to(device=device, dtype=dtype),
            negative_pooled_prompt_embeds=req.negative_pooled_prompt_embeds[None].to(device=device, dtype=dtype))
        init_image, mask, masked_image, mask_latent = pipe._preprocess_image_mask(
            req.image[None].to(device=device), req.mask_image[None].to(device=device), None, H, W)
        latents, = pipe.prepare_latents(1, pipe.vae.config.latent_channels, H, W, pe.dtype, device, gen, None,
                                        image=init_image, timestep=self.timesteps[:1], is_strength_max=True)  # draw 1
        mask, masked_lat = pipe.prepare_mask_latents(mask, masked_image, 1, H, W, pe.dtype, device, gen, do_cfg,
                                                     _mask_latent=mask_latent)                               # draw 2
        with _seeded_global_rng(device, self._seed(req)):
            pose = pipe._pose_latents(req.pose_img[None].to(device=device, dtype=pe.dtype), pe.dtype)        # global
        proj_dim = int(ppe.shape[-1]) if pipe.text_encoder_2 is None else pipe.text_encoder_2.config.projection_dim
        size = (latents.shape[-2] * pipe.vae_scale_factor, latents.shape[-1] * pipe.vae_scale_factor)
        add_time_ids, add_neg_time_ids = pipe._get_add_time_ids(size, (0, 0), size, 6.0, 2.5, size, (0, 0), size,
                                                                dtype=pe.dtype, text_encoder_projection_dim=proj_dim)
        add_text = ppe
        if do_cfg:
            pe, add_text = torch.cat([npe, pe]), torch.cat([nppe, ppe])
            add_time_ids = torch.cat([add_neg_time_ids, add_time_ids])
        return dict(latents=latents, mask=mask[:1], masked_image_latents=masked_lat[:1], pose_latents=pose,
                    prompt_embeds=pe.to(device), add_text_embeds=add_text.to(device), add_time_ids=add_time_ids.to(device))

    def _seed(self, req):
        return req.seed if req.seed is not None else self.seed

    def _admit(self):
        """Waiting requests, in ticket order, into the free slots, lowest slot first."""
        free = [s for s, e in enumerate(self.slots) if e is None]
        if not free or not self.waiting:
            return
        if not getattr(self, "_configured", False):
            self._configure()
        device, dtype = self.pipe._execution_device, self.pipe.unet.dtype
        for s in free:
            if not self.waiting:
                break
            req = self.waiting.popleft()
            g = self._garment(req, device, dtype)
            seed = self._seed(req)
            gen = torch.Generator(device).manual_seed(seed) if seed is not None else None
            prep = self._prepare_request(req, gen)
            page = None if self.garment_kv_bytes is None else self._pin_page(req.garment_id, g)
            self.den.admit(s, cloth_latents=g["latents"], image_embeds=g["image_embeds"],
                           text_embeds_cloth=g["text_embeds_cloth"], page=page, **prep)
            self.slots[s] = dict(req=req, gen=gen, step=0, page=page)
            self.stats["admitted"] += 1

    def _pin_page(self, gid, g):
        """Pool mode: the page holding garment `gid`, pinned for one more slot. A miss fills a free page, else the least
        recently admitted unpinned one (one exists: a free slot means at most slots - 1 pinned pages, and P >= slots)."""
        p = self.page_of.get(gid)
        if p is not None:
            self.page_of.move_to_end(gid)
            self.stats["garment_page_hits"] += 1
        else:
            if self.free_pages:
                p = self.free_pages.pop(0)
            else:
                victim = next(k for k, q in self.page_of.items() if self.pins[q] == 0)
                p = self.page_of.pop(victim)
                self.stats["garment_page_evictions"] += 1
            self.den.fill_page(p, g["latents"], g["text_embeds_cloth"])
            self.page_of[gid] = p
            self.stats["garment_page_fills"] += 1
        self.pins[p] += 1
        return p

    def _decode(self, latents):
        if self.output_type == "latent":
            return latents
        return self.pipe._postprocess(self.pipe._decode_latents(latents), self.output_type)

    @torch.no_grad()
    def step(self, use_graph=True):
        """Admits, runs one denoise step, decodes and frees the slots that finished. Returns {ticket: image}."""
        self._admit()
        active = [s for s, e in enumerate(self.slots) if e is not None]
        if not active:
            return {}
        from .denoise import variance_noise
        den = self.den
        device = self.pipe._execution_device
        noises = {}
        for s in active:
            e = self.slots[s]
            n = variance_noise(den, e["step"], (1, 4, *self.latent_size), e["gen"], device, den.latents.dtype)
            if n is not None:
                noises[s] = n
        latents = den.step([None if e is None else e["step"] for e in self.slots], noises,
                           use_graph=use_graph and getattr(self.pipe, "use_cuda_graph", True))
        self.stats["steps"] += 1
        self.stats["slot_steps"] += len(active)
        done = []
        for s in active:
            self.slots[s]["step"] += 1
            if self.slots[s]["step"] == self.T:
                done.append(s)
        if not done:
            self.last_latents = {}
            return {}
        final = latents[done].clone()
        tickets = [self.slots[s]["req"].ticket for s in done]
        self.last_latents = dict(zip(tickets, final))
        images = self._decode(final)
        for s in done:
            den.release(s)
            if self.slots[s]["page"] is not None:      # the page stays resident as a cache entry
                self.pins[self.slots[s]["page"]] -= 1
            self.slots[s] = None
        self.stats["images"] += len(done)
        return {t: images[i] for i, t in enumerate(tickets)}

    def run(self, use_graph=True):
        """Steps until every submitted request is finished; returns {ticket: image}."""
        out = {}
        while self.pending():
            out.update(self.step(use_graph=use_graph))
        return out
