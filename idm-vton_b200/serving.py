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
import contextlib
import copy
import dataclasses
from typing import Any, Hashable, Optional

import torch

from .denoise import GarmentKVCache
from .engine import active_freeu


@dataclasses.dataclass
class TryOnRequest:
    """One person x one garment. Tensors follow the keyword set of inference.py:397-414 for a batch of 1.

    A photo request passes image=None and `photo`: a full-resolution photo of any size (PIL RGB, or uint8 [H, W, 3] on
    the CPU or the GPU) or a photo.PreparedPhoto entry (not resampled again). The server crops it to its aspect,
    resamples it to its height x width with Pillow's filter (photo.prepare_photos) and pastes the output back into the
    photo (photo.paste_back, `paste`: "crop" replaces the whole box, "mask" only the masked pixels). mask_image and
    pose_img may then come at the server size, as below, or at photo size (mask: PIL "L" / "1" or uint8 / bool [H, W];
    pose: PIL RGB or uint8 [H, W, 3]); with a PreparedPhoto that holds them they may be None. The result is at photo
    size: a PIL image ("pil"), a uint8 [H, W, 3] CUDA tensor ("pt"), a uint8 [H, W, 3] numpy array ("np"), or the
    final latents ("latent").

    Garment side, needed the first time a garment_id is seen and ignored afterwards: its image as `cloth` and
    `ip_adapter_image`, or as `garment_photo` (a PIL image of any mode or a uint8 [H, W, 3] tensor, any size, on the CPU
    or the GPU; the server resizes it and makes both tensors as the demo does: photo.prepare_garments); its text as
    `text_embeds_cloth`, or as `garment_description` (encoded once per garment with the demo's prompts: PERSON_PROMPT,
    GARMENT_PROMPT, NEGATIVE_PROMPT). A request without the four prompt embeddings uses the person prompt of its
    garment's description."""
    garment_id: Hashable
    image: Optional[torch.Tensor]       # [3,H,W] in [0,1]; None with `photo`
    mask_image: Any                     # [1,H,W]
    pose_img: Any                       # [3,H,W] in [-1,1]
    prompt_embeds: Optional[torch.Tensor] = None         # [77,2048]; the four: all given or all None
    negative_prompt_embeds: Optional[torch.Tensor] = None
    pooled_prompt_embeds: Optional[torch.Tensor] = None  # [1280]
    negative_pooled_prompt_embeds: Optional[torch.Tensor] = None
    # garment side (needed the first time a garment_id is seen; ignored afterwards)
    cloth: Optional[torch.Tensor] = None             # [3,H,W] in [-1,1]
    ip_adapter_image: Optional[torch.Tensor] = None  # [3,224,224] CLIP-preprocessed garment image
    text_embeds_cloth: Optional[torch.Tensor] = None  # [77,2048]
    ticket: Any = None
    seed: Optional[int] = None          # ContinuousTryOnServer: this request's generator (TryOnServer ignores it)
    sampling: Optional[Hashable] = None  # the name of the server's SamplingPreset; None: the server's default preset
    photo: Any = None                   # a full-resolution photo or a photo.PreparedPhoto (image=None then)
    paste: str = "crop"                 # photo requests: "crop" (the demo's paste-back) or "mask"
    garment_photo: Any = None           # instead of cloth and ip_adapter_image
    garment_description: Optional[str] = None  # instead of text_embeds_cloth (and of the prompt embeddings)


# The demo's prompts (gradio_demo/app.py:178-179, 193-194) for a garment description d: the person prompt
# PERSON_PROMPT + d with classifier-free guidance against NEGATIVE_PROMPT, the garment prompt GARMENT_PROMPT + d without.
PERSON_PROMPT = "model is wearing "
GARMENT_PROMPT = "a photo of "
NEGATIVE_PROMPT = "monochrome, lowres, bad anatomy, worst quality, low quality"
PROMPT_FIELDS = ("prompt_embeds", "negative_prompt_embeds", "pooled_prompt_embeds", "negative_pooled_prompt_embeds")


def encode_description(pipe, description, device=None):
    """The demo's two encode_prompt calls for a garment description: {the four PROMPT_FIELDS, text_embeds_cloth}, each
    without its batch dimension (the shapes of the TryOnRequest fields)."""
    pe, npe, ppe, nppe = pipe.encode_prompt(PERSON_PROMPT + description, device=device, num_images_per_prompt=1,
                                            do_classifier_free_guidance=True, negative_prompt=NEGATIVE_PROMPT)
    cloth = pipe.encode_prompt([GARMENT_PROMPT + description], device=device, num_images_per_prompt=1,
                               do_classifier_free_guidance=False, negative_prompt=[NEGATIVE_PROMPT])[0]
    return dict(prompt_embeds=pe[0], negative_prompt_embeds=npe[0], pooled_prompt_embeds=ppe[0],
                negative_pooled_prompt_embeds=nppe[0], text_embeds_cloth=cloth[0])


def _can_encode(pipe):
    """Whether encode_prompt can run: tokenizer_2 and text_encoder_2, and the first pair both or neither."""
    get = lambda n: getattr(pipe, n, None)  # noqa: E731
    return get("tokenizer_2") is not None and get("text_encoder_2") is not None and \
        (get("tokenizer") is None) == (get("text_encoder") is None)


def _has_garment_image(req):
    return req.cloth is not None or req.garment_photo is not None


def _derived_garment(req):
    """Whether the garment `req` brings is made by the server (a garment photo or a description)."""
    return req.garment_photo is not None or req.garment_description is not None


def _check_garment_request(req, pipe, source):
    """Submit-time checks of a request's garment and prompt fields (ValueError). source: the garment's entry (a dict)
    when it is encoded, the request that brought it when that request still waits, None when `req` brings it."""
    gid = req.garment_id
    if req.garment_photo is not None:
        if req.cloth is not None or req.ip_adapter_image is not None:
            raise ValueError("garment_photo replaces cloth and ip_adapter_image: give one or the other")
        from .photo import check_garment
        check_garment(req.garment_photo)
    if req.garment_description is not None:
        if req.text_embeds_cloth is not None:
            raise ValueError("garment_description replaces text_embeds_cloth: give one or the other")
        if not isinstance(req.garment_description, str):
            raise ValueError(f"garment_description must be a str, got {type(req.garment_description).__name__}")
        if not _can_encode(pipe):
            raise ValueError("garment_description needs a pipeline with its tokenizers and text encoders")
    given = sum(getattr(req, f) is not None for f in PROMPT_FIELDS)
    if given not in (0, len(PROMPT_FIELDS)):
        raise ValueError(f"give all four prompt embeddings {PROMPT_FIELDS} or none (got {given})")
    if source is None:
        if req.garment_photo is None and (req.cloth is None or req.ip_adapter_image is None):
            raise ValueError(f"garment {gid!r} is new: cloth and ip_adapter_image, or garment_photo, are required")
        if req.text_embeds_cloth is None and req.garment_description is None:
            raise ValueError(f"garment {gid!r} is new: text_embeds_cloth or garment_description is required")
        described = req.garment_description is not None
    else:
        described = "prompt_embeds" in source if isinstance(source, dict) else source.garment_description is not None
    if not given and not described:
        raise ValueError(f"the request has no prompt embeddings and garment {gid!r} has no garment_description to "
                         "make them from")


def _prompts(req, g):
    """The request's four prompt embeddings, or its garment's description-derived ones."""
    if req.prompt_embeds is not None:
        return [getattr(req, f) for f in PROMPT_FIELDS]
    return [g[f] for f in PROMPT_FIELDS]


class _GarmentFailed(Exception):
    """A garment made by the server (photo or description) could not be prepared; __cause__ is the error."""


def _prepare_garment_photos(photos, height, width):
    """(entries, failed): photo.prepare_garments of `photos` in one call. If that call raises, each photo is prepared
    on its own, and the ones that still raise come back in `failed` ({index: exception}, entry None). A library without
    the kernels raises (NotImplementedError)."""
    from .photo import prepare_garments
    if not photos:
        return [], {}
    try:
        return prepare_garments(photos, height, width), {}
    except NotImplementedError:
        raise
    except (ValueError, RuntimeError):
        entries, failed = [None] * len(photos), {}
        for i, p in enumerate(photos):
            try:
                entries[i] = prepare_garments([p], height, width)[0]
            except NotImplementedError:
                raise
            except (ValueError, RuntimeError) as exc:
                failed[i] = exc
        return entries, failed


@dataclasses.dataclass
class SamplingPreset:
    """How a request is denoised: the pipeline's `__call__` arguments of the same names. scheduler: a diffusers-style
    scheduler object (None: the pipeline's); the server steps a private copy of it."""
    scheduler: Any = None
    num_inference_steps: int = 30
    guidance_scale: float = 2.0
    strength: float = 1.0
    eta: float = 0.0
    guidance_rescale: float = 0.0


def _check_presets(presets, default_preset):
    """(presets, default name) of a server's `presets` / `default_preset` arguments: a non-empty dict of SamplingPreset;
    the default may be omitted when there is one preset."""
    presets = dict(presets)
    if not presets or not all(isinstance(p, SamplingPreset) for p in presets.values()):
        raise ValueError("presets must be a non-empty dict of name -> SamplingPreset")
    if default_preset is None and len(presets) == 1:
        default_preset = next(iter(presets))
    if default_preset not in presets:
        raise ValueError(f"default_preset {default_preset!r} is not one of the presets {list(presets)}")
    return presets, default_preset


def _preset_name(server, req):
    name = server.default_preset if req.sampling is None else req.sampling
    if name not in server.presets:
        raise ValueError(f"request names sampling preset {req.sampling!r}; the server has {list(server.presets)}")
    return name


def _private(scheduler):
    """A copy of `scheduler` whose set_timesteps leaves the original as it was: set_timesteps rebinds the attributes it
    sets, and the shared config and training tables are only read."""
    return copy.copy(scheduler)


@contextlib.contextmanager
def _scheduler_installed(pipe, scheduler):
    """pipe.scheduler = scheduler for the block (None: the pipeline's own), restored afterwards."""
    if scheduler is None:
        yield
        return
    old = pipe.scheduler
    pipe.scheduler = scheduler
    try:
        yield
    finally:
        pipe.scheduler = old


def _encode_garment(pipe, src, seed, device, dtype, prepared=None):
    """ONE posterior sample per garment, from a generator of its own (seeded with the server's seed): the per-request
    generator must see the same stream whether or not the garment was already known. prepared: the PreparedGarment of
    src.garment_photo (its cloth and CLIP pixels replace src's). A garment_description is encoded here, once: the
    entry then holds its text_embeds_cloth and the four person-prompt embeddings."""
    cloth = (src.cloth if prepared is None else prepared.cloth)[None].to(device=device, dtype=dtype)
    gen = torch.Generator(device).manual_seed(seed) if seed is not None else None
    latents = pipe._encode_vae_image(cloth, generator=gen)
    ip = src.ip_adapter_image if prepared is None else prepared.clip_pixels
    g = dict(latents=latents, ip_adapter_image=ip[None].to(device))
    if src.garment_description is None:
        g["text_embeds_cloth"] = src.text_embeds_cloth[None].to(device=device, dtype=dtype)
    else:
        emb = encode_description(pipe, src.garment_description, device)
        g["text_embeds_cloth"] = emb.pop("text_embeds_cloth")[None].to(device=device, dtype=dtype)
        g.update(emb)
    return g


def _check_photo_request(req, height, width):
    """Submit-time checks of a request with `photo` (ValueError): no `image` beside it, a supported photo, a mask and a
    pose at the server size or at the photo's, and a paste mode."""
    if req.photo is None:
        return
    from . import photo as P
    if req.image is not None:
        raise ValueError("a request with `photo` passes image=None: the server makes the image from the photo")
    if req.paste not in P.PASTE_MODES:
        raise ValueError(f"paste must be one of {P.PASTE_MODES}, got {req.paste!r}")
    P.check_photo(req.photo)
    size = P.photo_size(req.photo)
    prepared = req.photo if isinstance(req.photo, P.PreparedPhoto) else None
    if prepared is not None and tuple(prepared.image.shape[-2:]) != (height, width):
        raise ValueError(f"the photo was prepared at {tuple(prepared.image.shape[-2:])}, the server runs at "
                         f"{(height, width)}")
    if prepared is None:
        P.check_crop(size, height, width)
    for value, kind, check in ((req.mask_image, "mask", P.mask_size), (req.pose_img, "pose", P.pose_size)):
        if value is not None:
            check(value, size, height, width)
        elif prepared is None or getattr(prepared, kind) is None:
            raise ValueError(f"a photo request needs its {'mask_image' if kind == 'mask' else 'pose_img'} (at the "
                             "server's size or the photo's), or a PreparedPhoto that holds it")


def _prepare_photos(reqs, height, width, filter):
    """The PreparedPhoto of each photo request of `reqs` (None for the others), one resample call for all of them:
    photo-size masks and poses are resampled with the photo."""
    from . import photo as P
    idx = [i for i, r in enumerate(reqs) if r.photo is not None]
    out = [None] * len(reqs)
    if not idx:
        return out
    photo_size = lambda r, v, fn: v if v is not None and fn(v, P.photo_size(r.photo), height, width) == "photo" \
        else None  # noqa: E731
    entries = P.prepare_photos([reqs[i].photo for i in idx], height, width, filter=filter,
                               masks=[photo_size(reqs[i], reqs[i].mask_image, P.mask_size) for i in idx],
                               poses=[photo_size(reqs[i], reqs[i].pose_img, P.pose_size) for i in idx])
    for i, e in zip(idx, entries):
        out[i] = e
    return out


def _prepare_photos_or_drop(reqs, height, width, filter):
    """(entries, failed): _prepare_photos of `reqs` in one call. If that call raises, each photo request is prepared
    on its own, and the ones that still raise come back in `failed` ({index: exception}, no entry), so one bad request
    cannot stop the server. A library without the photo kernels raises (NotImplementedError) for all of them."""
    try:
        return _prepare_photos(reqs, height, width, filter), {}
    except NotImplementedError:
        raise
    except (ValueError, RuntimeError):
        entries, failed = [None] * len(reqs), {}
        for i, r in enumerate(reqs):
            if r.photo is None:
                continue
            try:
                entries[i] = _prepare_photos([r], height, width, filter)[0]
            except NotImplementedError:
                raise
            except (ValueError, RuntimeError) as exc:
                failed[i] = exc
        return entries, failed


def _person_inputs(req, entry):
    """(image [3,H,W], mask [1,H,W], pose [3,H,W]) of a request at the server size: its own tensors, or for a photo
    request the prepared crop, with the resampled mask / pose where they came at photo size (photo.mask_size and
    photo.pose_size decide which size a mask or pose is, here as at submit)."""
    if entry is None:
        return req.image, req.mask_image, req.pose_img
    from . import photo as P
    h, w = entry.image.shape[-2:]
    server = lambda v, fn: v if v is not None and fn(v, entry.size, h, w) == "server" else None  # noqa: E731
    mask, pose = server(req.mask_image, P.mask_size), server(req.pose_img, P.pose_size)
    return entry.image, entry.mask if mask is None else mask, entry.pose if pose is None else pose


def _photo_result(full, output_type):
    if output_type == "pt":
        return full
    a = full.cpu().numpy()
    if output_type == "np":
        return a
    import PIL.Image
    return PIL.Image.fromarray(a)


def _decode_with_photos(pipe, output_type, latents, entries, reqs):
    """Images of requests that finish together, from their final latents (output_type is not "latent"): one VAE decode;
    rows without a photo get the pipeline's own post-processing of their rows (the bits they get without photos);
    photo rows get the uint8 output the pipeline's "pil" is made of, pasted back into their photos in one launch."""
    from . import lib as L
    from . import photo as P
    decoded = pipe._decode_latents(latents)
    out = [None] * len(entries)
    plain = [i for i, e in enumerate(entries) if e is None]
    photo = [i for i, e in enumerate(entries) if e is not None]
    if plain:
        imgs = pipe._postprocess(decoded if not photo else decoded[plain], output_type)
        for j, i in enumerate(plain):
            out[i] = imgs[j]
    _, u8 = L.postprocess_image(decoded if not plain else decoded[photo], want_pt=False, want_u8=True)
    full = P.paste_back([entries[i] for i in photo], u8, [reqs[i].paste for i in photo],
                        masks=[_person_inputs(reqs[i], entries[i])[1] for i in photo])
    for j, i in enumerate(photo):
        out[i] = _photo_result(full[j], output_type)
    return out


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
    """Batch mode: requests that wear the same garment and use the same sampling preset run as one pipeline call.
    presets: {name: SamplingPreset} (a request picks one by `sampling`; default_preset when it names none); each batch
    calls the pipeline with its preset's arguments, its scheduler (a private copy) installed for the call. None: one
    preset from num_inference_steps and guidance_scale with the pipeline's scheduler.
    Photo requests (TryOnRequest.photo) whose preparation fails are dropped from their batch, which still runs; their
    tickets map to the exception in `failed`. A garment made from a garment_photo or a garment_description is prepared
    when its first batch runs; if that fails, every waiting request of its garment_id goes to `failed`."""

    def __init__(self, pipe, height=1024, width=768, num_inference_steps=30, guidance_scale=2.0, max_batch=8, seed=None,
                 garment_cache_bytes=40 << 30, output_type="pt", presets=None, default_preset=None, photo_filter="bicubic"):
        from .photo import _check_filter
        _check_filter(photo_filter)
        self.photo_filter = photo_filter
        self.pipe = pipe
        self.height, self.width = height, width
        self.num_inference_steps, self.guidance_scale = num_inference_steps, guidance_scale
        self.max_batch = max_batch
        self.seed = seed
        self.output_type = output_type
        if presets is None:
            self.presets, self.default_preset = {None: None}, None       # built from the attributes at each batch
        else:
            self.presets, self.default_preset = _check_presets(presets, default_preset)
        self._schedulers = {n: None if p is None or p.scheduler is None else _private(p.scheduler)
                            for n, p in self.presets.items()}
        self.queue = collections.OrderedDict()      # (garment_id, preset) -> deque of requests (arrival order)
        self.garments = {}                          # garment_id -> dict(latents, ip_adapter_image, text_embeds_cloth)
        self._next_ticket = 0
        self.stats = collections.Counter()
        self.failed = {}                             # ticket -> exception: photo requests whose preparation failed
        if garment_cache_bytes:
            pipe.garment_cache = GarmentKVCache(garment_cache_bytes)

    # ---------------------------------------------------------------------------------------------
    def submit(self, req: TryOnRequest):
        name = _preset_name(self, req)
        _check_photo_request(req, self.height, self.width)
        g = self.garments.get(req.garment_id)
        _check_garment_request(req, self.pipe, g if g is not None else self._pending_source(req.garment_id))
        req.ticket = self._next_ticket
        self._next_ticket += 1
        self.queue.setdefault((req.garment_id, name), collections.deque()).append(req)
        return req.ticket

    def pending(self):
        return sum(len(q) for q in self.queue.values())

    def _next_batch(self):
        """Oldest waiting request decides the garment and the preset; up to max_batch requests of both go together."""
        key = min(self.queue, key=lambda k: self.queue[k][0].ticket)
        q = self.queue[key]
        batch = [q.popleft() for _ in range(min(self.max_batch, len(q)))]
        if not q:
            del self.queue[key]
        return key, batch

    def _preset(self, name):
        p = self.presets[name]
        return SamplingPreset(None, self.num_inference_steps, self.guidance_scale) if p is None else p

    def _pending_source(self, gid, extra=()):
        """The waiting request (of `extra` or the queue) that brought garment `gid`: the first one with its image."""
        cands = [r for r in extra if _has_garment_image(r)]
        cands += [r for (g, _), q in self.queue.items() if g == gid for r in q if _has_garment_image(r)]
        return min(cands, key=lambda r: r.ticket) if cands else None

    def _garment(self, gid, batch, device, dtype):
        """The garment's entry, encoded on first use. A garment made from a photo or a description that fails raises
        _GarmentFailed."""
        g = self.garments.get(gid)
        if g is None:
            src = self._pending_source(gid, batch)
            try:
                prepared = None
                if src.garment_photo is not None:
                    entries, failed = _prepare_garment_photos([src.garment_photo], self.height, self.width)
                    if failed:
                        raise failed[0]
                    prepared = entries[0]
                    self.stats["garment_photos_prepared"] += 1
                g = _encode_garment(self.pipe, src, self.seed, device, dtype, prepared)
            except NotImplementedError:
                raise
            except (ValueError, RuntimeError) as exc:
                if not _derived_garment(src):
                    raise
                raise _GarmentFailed(f"garment {gid!r} could not be prepared") from exc
            self.stats["descriptions_encoded"] += src.garment_description is not None
            self.garments[gid] = g
            self.stats["garments_encoded"] += 1
        return g

    def _drop_garment(self, gid, batch, exc):
        """Every waiting request of garment `gid` (`batch` and the queue) fails with `exc`; the id is unknown again."""
        dropped = list(batch)
        for key in [k for k in self.queue if k[0] == gid]:
            dropped += self.queue.pop(key)
        for r in dropped:
            self.failed[r.ticket] = exc
        self.stats["failed"] += len(dropped)

    @torch.no_grad()
    def step(self):
        """Runs ONE batch; returns {ticket: image}."""
        if not self.queue:
            return {}
        (gid, name), batch = self._next_batch()
        preset = self._preset(name)
        pipe = self.pipe
        device = pipe._execution_device
        dtype = pipe.unet.dtype
        try:
            g = self._garment(gid, batch, device, dtype)
        except _GarmentFailed as exc:       # the garment's requests are dropped; the server goes on
            self._drop_garment(gid, batch, exc.__cause__)
            return {}
        gen = torch.Generator(device).manual_seed(self.seed) if self.seed is not None else None
        stack = lambda name, dt=None: torch.stack([getattr(r, name) for r in batch]).to(device=device, dtype=dt)  # noqa: E731
        prompts = [_prompts(r, g) for r in batch]
        # a request's own tensors may be on the host, a garment's derived ones are on the device
        prompt = lambda j: torch.stack([p[j].to(device=device, dtype=dtype) for p in prompts])  # noqa: E731
        entries, failed = _prepare_photos_or_drop(batch, self.height, self.width, self.photo_filter)
        if failed:            # dropped from the batch; the rest of it runs
            for i, exc in failed.items():
                self.failed[batch[i].ticket] = exc
            self.stats["failed"] += len(failed)
            batch = [r for i, r in enumerate(batch) if i not in failed]
            entries = [e for i, e in enumerate(entries) if i not in failed]
            if not batch:
                return {}
        photos = any(e is not None for e in entries)
        if photos:            # the photo requests' crops (one resample launch) beside the others' tensors
            person = [_person_inputs(r, e) for r, e in zip(batch, entries)]
            person = {k: torch.stack([p[j].to(device=device) for p in person]) for j, k in enumerate(("image",
                                                                                                      "mask_image",
                                                                                                      "pose_img"))}
            person["pose_img"] = person["pose_img"].to(dtype)
        else:
            person = dict(image=stack("image"), mask_image=stack("mask_image"), pose_img=stack("pose_img", dtype))
        # photo rows are decoded here, after the call, so that they can be pasted back (output_type "latent" skips it)
        out_type = "latent" if photos else self.output_type
        # eta and guidance_rescale are passed only when a preset sets them (the pipeline's defaults otherwise)
        extra = {k: getattr(preset, k) for k in ("eta", "guidance_rescale") if getattr(preset, k)}
        # the pose latents' sample comes from the global generator: seeded around the call (_seeded_global_rng), so a
        # seeded server is reproducible
        with _scheduler_installed(pipe, self._schedulers[name]), _seeded_global_rng(device, self.seed):
            images = pipe(prompt_embeds=prompt(0), negative_prompt_embeds=prompt(1), pooled_prompt_embeds=prompt(2),
                          negative_pooled_prompt_embeds=prompt(3),
                          num_inference_steps=preset.num_inference_steps, generator=gen, strength=preset.strength,
                          pose_img=person["pose_img"], text_embeds_cloth=g["text_embeds_cloth"], cloth=g["latents"],
                          mask_image=person["mask_image"], image=person["image"], height=self.height,
                          width=self.width, ip_adapter_image=g["ip_adapter_image"],
                          guidance_scale=preset.guidance_scale, output_type=out_type, garment_keys=[gid], **extra)[0]
        if photos:
            latents = pipe._last_latents
            if self.output_type == "latent":
                images = [latents[i] if e is not None else images[i] for i, e in enumerate(entries)]
            else:
                images = _decode_with_photos(pipe, self.output_type, latents, entries, batch)
        self.stats["batches"] += 1
        self.stats["images"] += len(batch)
        return {r.ticket: images[i] for i, r in enumerate(batch)}

    def run(self):
        """Drains the queue; returns {ticket: image}."""
        out = {}
        while self.queue:
            out.update(self.step())
        return out


# ContinuousTryOnServer.stats of the garment K/V pool's host tier
HOST_STATS = ("garment_host_hits", "garment_host_writes", "garment_host_skipped", "garment_host_evictions",
              "garment_rows_streamed", "garment_bytes_streamed")


def _freeu(pipe):
    """The FreeU values the pipeline's try-on UNet runs with (enable_freeu, all four non-zero), or None."""
    return active_freeu(getattr(pipe.unet, "freeu", None))


class ContinuousTryOnServer:
    """Continuous batching: requests join and leave the denoise batch at every step (denoise.SlotDenoiser).

    The server has `slots` slots. Each `step()` admits waiting requests into free slots (lowest slot first, in ticket
    order), replays ONE denoise step in which every occupied slot advances its own request by one step, then VAE-decodes
    the requests that finished (one decode for all of them) and frees their slots. A request therefore waits for a free
    slot, not for a whole batch, and a batch that is not full fills up at the next step.

    One person size (height x width); the garment must have the same latent size. Garments are VAE-encoded once per
    garment_id exactly as TryOnServer does.

    Sampling presets: presets=None runs every request with the pipeline's scheduler, num_inference_steps, guidance_scale
    and eta at strength 1. presets={name: SamplingPreset} lets each request pick one by `sampling` (default_preset when
    it names none): its own scheduler (a private copy per preset: one preset's set_timesteps touches no other preset
    and not pipe.scheduler), step count, strength, guidance scale, eta and, with DDPM, guidance rescale. Every preset's
    plan is built at the first step. One preset without guidance rescale runs the per-kind step kernels; two or more,
    or guidance rescale, run SlotDenoiser.configure_presets and the mixed-kind step kernel, where each request gets the
    bits it gets from a one-preset server. A request retires after its own preset's number of steps.

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
      * garment_kv_host_bytes=M beside garment_kv_bytes (pool mode with a host tier): Q = M // page_bytes more pages in
        page-locked host memory, in the pool's format (denoise.HostGarmentKV), with an LRU of their own. Admission looks
        a garment up on the device (pin the page), then on the host (the slot streams host page q, pinned there: each
        step's row is copied into a ring of two device rows per slot beside the step before, SlotDenoiser), then fills
        a device page and writes it through to a host page on a side stream (skipped and counted when every host page
        is pinned). A device page whose write-through is in flight is refilled only after it, on the device. A host
        hit is not copied back to a device page. Refused before any launch: garment_kv_host_bytes without
        garment_kv_bytes and a host budget below one page (ValueError), and a failed page-lock (RuntimeError naming the
        bytes). close() unregisters the host memory. `stats` adds garment_host_hits, garment_host_writes,
        garment_host_skipped, garment_host_evictions, garment_rows_streamed and garment_bytes_streamed.

    RNG: each request owns a generator seeded with `req.seed` (the server's seed when None; unseeded when both are None)
    and draws in the order the pipeline draws for a batch of one: the initial noise, the masked image's VAE sample, the
    pose sample from the global generator (forked and seeded with the same seed, as TryOnServer does), then the variance
    noise of every step whose scheduler step draws one. A request's result is then independent of arrival order, slot
    and neighbours (at a fixed number of slots): its final latents always, its image when it finishes at a step of its
    own (requests finishing at the same step share one VAE decode).
    `eta`: DDIM's eta, as the pipeline's `__call__` takes it (0 = deterministic DDIM, 1 = DDPM-like variance).
    Pool mode with presets: a page holds T_max (the largest step count of the presets) steps, and pages are keyed by
    (garment_id, the preset's timesteps), so presets with the same timesteps share a garment's page.
    Refused, before any launch: guidance_rescale without presets (not a parameter here) and with a scheduler other
    than DDPM (NotImplementedError); presets with guidance_scale <= 1 beside presets with CFG (ValueError); schedulers
    other than DDPM / DDIM / Euler / DPM-Solver++; a library without the per-slot step kernels, the mixed-kind step
    kernel (b200vton_cfg_step_mixed_rows) when presets need it, or, in pool mode, b200vton_attention_rows
    (NotImplementedError naming the symbol). An unknown preset name is refused at submit (ValueError).
    Photo requests (TryOnRequest.photo) are prepared at admission; one whose preparation fails is dropped from the queue
    without taking a slot, and its ticket maps to the exception in `failed`. The new garments of an admission made from
    a garment_photo or a garment_description are prepared there, their photos in one prepare_garments call; a garment
    that fails takes every waiting request of its garment_id to `failed`."""

    def __init__(self, pipe, height=1024, width=768, slots=4, num_inference_steps=30, guidance_scale=2.0, seed=None,
                 output_type="pt", eta=0.0, garment_kv_bytes=None, presets=None, default_preset=None,
                 photo_filter="bicubic", garment_kv_host_bytes=None):
        from .photo import _check_filter
        _check_filter(photo_filter)
        if garment_kv_host_bytes is not None and garment_kv_bytes is None:
            raise ValueError("garment_kv_host_bytes is a host tier of the garment K/V pool: it needs garment_kv_bytes")
        self.photo_filter = photo_filter
        self.pipe = pipe
        self.height, self.width = height, width
        self.S = int(slots)
        self.num_inference_steps, self.guidance_scale = num_inference_steps, guidance_scale
        self.seed = seed
        self.output_type = output_type
        self.eta = float(eta)                        # DDIM's eta (the pipeline's `eta`; other schedulers ignore it)
        self.guidance_rescale = 0.0
        if presets is None:
            self.presets, self.default_preset = {None: None}, None       # built from the attributes at configure
        else:
            self.presets, self.default_preset = _check_presets(presets, default_preset)
        # two or more presets, or guidance rescale: the mixed-kind step
        self.mixed = len(self.presets) > 1 or any(p is not None and p.guidance_rescale > 0 for p in self.presets.values())
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
        self.garment_kv_host_bytes = None if garment_kv_host_bytes is None else int(garment_kv_host_bytes)
        self.host_page_of = collections.OrderedDict()    # host tier: key -> host page, least recently used first
        self.host_pins = collections.Counter()           # host tier: host page -> slots streaming from it
        self.free_host_pages = []
        self.last_latents = {}                       # ticket -> final latents of the requests the last step() finished
        self._next_ticket = 0
        self.stats = collections.Counter()
        self.failed = {}                             # ticket -> exception: requests whose photo or garment failed
        self._prepared_garments = {}                 # garment_id -> PreparedGarment made at this admission

    # ---------------------------------------------------------------------------------------------
    def submit(self, req: TryOnRequest):
        _preset_name(self, req)
        _check_photo_request(req, self.height, self.width)
        g = self.garments.get(req.garment_id)
        source = g if g is not None else self._pending_source(req.garment_id)
        _check_garment_request(req, self.pipe, source)
        if source is None and req.garment_photo is None:       # a garment photo is resized to the server's size
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
    def _make_denoiser(self, pages=None, **host):
        from .denoise import SlotDenoiser
        return SlotDenoiser(self.pipe.unet.engine(), self.pipe.unet_encoder.engine(), self.S, pages=pages, **host)

    def _new_pool(self, T):
        """Pool mode: a denoiser with a pool of pages of T rows and, with garment_kv_host_bytes, a host tier; every
        refusal comes first."""
        P, Q = self._pages(T), self._host_pages(T)
        self.den = self._make_denoiser(pages=P) if Q is None else self._make_denoiser(pages=P, host_pages=Q)
        self._reset_pages(P, Q)
        if Q is not None:                            # the host tier's counters, shown from the first admission
            self.stats.update(dict.fromkeys(HOST_STATS, 0))

    def _drop_denoiser(self):
        """Drops the denoiser; its host tier's memory is unregistered first."""
        release = getattr(self.den, "release_host", None)
        if release is not None:
            release()
        self.den = None

    def close(self):
        """Releases the garment K/V pool and unregisters the host tier's page-locked memory. The server stays usable:
        the next admission configures it again (with empty pages). Refused while requests run."""
        if any(e is not None for e in self.slots):
            raise RuntimeError("close() while requests run in slots")
        self._drop_denoiser()
        self._configured = False
        self._reset_pages(0)

    def page_bytes(self, T=None):
        """Pool mode: bytes of one garment's page, the hoisted K/V of all T steps at Bg = 1 (from the shapes). T defaults
        to the step count of the run, or with presets to the largest one after strength (T_max)."""
        from .denoise import garment_kv_bytes_per_step
        if T is None:
            T = max(self.num_inference_steps if p is None else
                    min(int(p.num_inference_steps * p.strength), p.num_inference_steps) for p in self.presets.values())
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

    def _host_pages(self, T):
        """Host tier: the number of pages its budget holds (None without a host tier); refuses less than one."""
        if self.garment_kv_host_bytes is None:
            return None
        page = self.page_bytes(T)
        Q = self.garment_kv_host_bytes // page
        if Q < 1:
            raise ValueError(f"garment_kv_host_bytes={self.garment_kv_host_bytes} holds no garment K/V page of {page} "
                             f"bytes ({page / 1e9:.2f} GB: {T} steps at latent size {self.latent_size}); the host tier "
                             "needs at least one page")
        return Q

    def _reset_pages(self, P, Q=None):
        self.page_of.clear()
        self.pins.clear()
        self.free_pages = list(range(P))
        self.host_page_of.clear()
        self.host_pins.clear()
        self.free_host_pages = list(range(Q or 0))

    def _preset(self, name):
        p = self.presets[name]
        return SamplingPreset(None, self.num_inference_steps, self.guidance_scale, 1.0, self.eta) if p is None else p

    def _run_timesteps(self, name):
        """The pipeline's own timestep selection for preset `name` (its scheduler installed: retrieve_timesteps, then
        get_timesteps at the preset's strength)."""
        from .pipeline import retrieve_timesteps
        pipe, p = self.pipe, self._preset(name)
        with _scheduler_installed(pipe, self._schedulers[name]):
            timesteps, n = retrieve_timesteps(pipe.scheduler, p.num_inference_steps, pipe._execution_device)
            timesteps, n = pipe.get_timesteps(n, p.strength, pipe._execution_device)
        if n < 1:
            raise ValueError(f"sampling preset {name!r}: strength {p.strength} at {p.num_inference_steps} steps leaves "
                             f"{n} steps")
        return timesteps

    def _configure(self):
        """Timesteps and per-step tables of every preset (the pipeline's own timestep selection); checks every refusal
        before the first launch."""
        pipe = self.pipe
        # private schedulers (presets given; the pipeline's own without presets)
        self._schedulers = {n: None if p is None else _private(pipe.scheduler if p.scheduler is None else p.scheduler)
                            for n, p in self.presets.items()}
        if self.mixed:
            return self._configure_presets()
        name = next(iter(self.presets))
        p = self._preset(name)
        pipe._guidance_scale = p.guidance_scale
        timesteps = self._run_timesteps(name)
        self.timesteps = timesteps
        self._timesteps = {name: timesteps}
        if self.den is None:
            if self.garment_kv_bytes is None:
                self.den = self._make_denoiser()
            else:
                self._new_pool(len(timesteps))
        self.den.configure(self._schedulers[name] or pipe.scheduler, timesteps, *self.latent_size,
                           guidance_scale=p.guidance_scale, do_cfg=pipe.do_classifier_free_guidance, eta=p.eta,
                           guidance_rescale=self.guidance_rescale)
        self.T = self.den.T
        self._configured = True

    def _configure_presets(self):
        """The mixed-kind path: one StepPlan per preset, refusals first."""
        from .denoise import check_guidance_rescale, scheduler_kind, step_plan
        pipe = self.pipe
        for name, p in self.presets.items():
            scheduler_kind(self._schedulers[name])
            check_guidance_rescale(self._schedulers[name], p.guidance_rescale)
        if len({p.guidance_scale > 1 for p in self.presets.values()}) > 1:
            raise ValueError("sampling presets with guidance_scale <= 1 (no classifier-free guidance) cannot share a "
                             "server with presets that use it: " +
                             ", ".join(f"{n!r}: {p.guidance_scale}" for n, p in self.presets.items()))
        pipe._guidance_scale = self.presets[self.default_preset].guidance_scale
        do_cfg = pipe.do_classifier_free_guidance
        self._timesteps = {n: self._run_timesteps(n) for n in self.presets}
        self._plan_index = {n: j for j, n in enumerate(self.presets)}
        self.plans = [step_plan(self._schedulers[n], self._timesteps[n], p.guidance_scale,
                                p.guidance_rescale if do_cfg else 0.0, p.eta) for n, p in self.presets.items()]
        T_max = max(plan.T for plan in self.plans)
        if self.den is None:
            if self.garment_kv_bytes is None:
                self.den = self._make_denoiser()
            else:
                self._new_pool(T_max)
        self.den.configure_presets(self.plans, *self.latent_size, do_cfg=do_cfg)
        self.T = T_max
        self._configured = True

    def _pending_source(self, gid):
        """The waiting request that brought garment `gid`: the first one with its image."""
        return next((r for r in self.waiting if r.garment_id == gid and _has_garment_image(r)), None)

    def _garment(self, req, device, dtype):
        """The garment's entry, encoded on first use (with the PreparedGarment of this admission when it has a photo).
        A garment made from a photo or a description that fails raises _GarmentFailed."""
        g = self.garments.get(req.garment_id)
        if g is None:
            src = req if _has_garment_image(req) else self._pending_source(req.garment_id)
            try:
                prepared = self._prepared_garments.pop(req.garment_id, None)
                if prepared is None and src.garment_photo is not None:
                    entries, failed = _prepare_garment_photos([src.garment_photo], self.height, self.width)
                    if failed:
                        raise failed[0]
                    prepared = entries[0]
                    self.stats["garment_photos_prepared"] += 1
                g = _encode_garment(self.pipe, src, self.seed, device, dtype, prepared)
                emb = self.pipe.prepare_ip_adapter_image_embeds(g["ip_adapter_image"], device, 1)
                g["image_embeds"] = self.pipe.unet.encoder_hid_proj(emb).to(dtype)         # Resampler, once per garment
            except NotImplementedError:
                raise
            except (ValueError, RuntimeError) as exc:
                if not _derived_garment(src):
                    raise
                raise _GarmentFailed(f"garment {req.garment_id!r} could not be prepared") from exc
            self.stats["descriptions_encoded"] += src.garment_description is not None
            self.garments[req.garment_id] = g
            self.stats["garments_encoded"] += 1
        return g

    def _encode_new_garments(self, heads, device, dtype):
        """Encodes the new garments of `heads` that the server makes itself (a photo or a description), their photos
        in one prepare_garments call. A garment that fails takes every waiting request of its id into `failed`, and the
        id is unknown again. Returns whether any was dropped (the heads changed)."""
        new = {}
        for r in heads:
            if r.garment_id not in self.garments and r.garment_id not in new:
                src = self._pending_source(r.garment_id)
                if src is not None and _derived_garment(src):
                    new[r.garment_id] = src
        photo = [gid for gid, src in new.items() if src.garment_photo is not None]
        entries, failed = _prepare_garment_photos([new[gid].garment_photo for gid in photo], self.height, self.width)
        dropped = {photo[j]: exc for j, exc in failed.items()}
        for gid, e in zip(photo, entries):
            if e is not None:
                self._prepared_garments[gid] = e
                self.stats["garment_photos_prepared"] += 1
        for gid, src in new.items():
            if gid not in dropped:
                try:
                    self._garment(src, device, dtype)
                except _GarmentFailed as exc:
                    dropped[gid] = exc.__cause__
        for gid, exc in dropped.items():
            self._prepared_garments.pop(gid, None)
            keep = collections.deque()
            for r in self.waiting:
                if r.garment_id == gid:
                    self.failed[r.ticket] = exc
                    self.stats["failed"] += 1
                else:
                    keep.append(r)
            self.waiting = keep
        return bool(dropped)

    def _prepare_request(self, req, gen, entry=None):
        """The pipeline's own preparation of one person (batch 1, the request's preset and its scheduler installed):
        pre-processing, initial latents (with strength < 1 the image's VAE sample, then the noise, added to it at the
        first timestep), mask and masked-image latents, pose latents, prompt and added-condition embeddings — drawing
        from `gen` in the pipeline's order. entry: the request's PreparedPhoto (photo requests). Returns the keyword
        arguments of SlotDenoiser.admit except the garment's."""
        name = _preset_name(self, req)
        with _scheduler_installed(self.pipe, self._schedulers[name]):
            return self._prepare_with(req, gen, self._preset(name).strength, self._timesteps[name], entry)

    def _prepare_with(self, req, gen, strength, timesteps, entry=None):
        pipe = self.pipe
        device, dtype = pipe._execution_device, pipe.unet.dtype
        do_cfg = pipe.do_classifier_free_guidance
        H, W = self.height, self.width
        prompts = [p[None].to(device=device, dtype=dtype) for p in _prompts(req, self.garments.get(req.garment_id))]
        pe, npe, ppe, nppe = pipe.encode_prompt(
            prompt=None, device=device, num_images_per_prompt=1, do_classifier_free_guidance=do_cfg,
            prompt_embeds=prompts[0], negative_prompt_embeds=prompts[1], pooled_prompt_embeds=prompts[2],
            negative_pooled_prompt_embeds=prompts[3])
        image, mask_image, pose_img = _person_inputs(req, entry)
        init_image, mask, masked_image, mask_latent = pipe._preprocess_image_mask(
            image[None].to(device=device), mask_image[None].to(device=device), None, H, W)
        latents, = pipe.prepare_latents(1, pipe.vae.config.latent_channels, H, W, pe.dtype, device, gen, None,
                                        image=init_image, timestep=timesteps[:1],
                                        is_strength_max=strength == 1.0)                                     # draw 1
        mask, masked_lat = pipe.prepare_mask_latents(mask, masked_image, 1, H, W, pe.dtype, device, gen, do_cfg,
                                                     _mask_latent=mask_latent)                               # draw 2
        with _seeded_global_rng(device, self._seed(req)):
            pose = pipe._pose_latents(pose_img[None].to(device=device, dtype=pe.dtype), pe.dtype)            # global
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
        fmt = getattr(self.pipe.unet, "garment_kv_precision", "fp16")
        if getattr(self, "_configured", False) and fmt != self._kv_format:
            # the pipe's garment K/V precision changed: the pool, its page count and the page table are in the old format
            if any(e is not None for e in self.slots):
                raise RuntimeError(f"the pipeline's garment K/V precision changed to {fmt!r} while requests run in "
                                   f"{self._kv_format!r}: change it when the server is idle")
            self._drop_denoiser()
            self._configured = False
        if not getattr(self, "_configured", False):
            self._configure()
            self._kv_format = fmt
            self._freeu = _freeu(self.pipe)
        device, dtype = self.pipe._execution_device, self.pipe.unet.dtype
        while free and self.waiting:       # again when a dropped request left a slot free
            n = min(len(free), len(self.waiting))
            heads = [self.waiting[i] for i in range(n)]
            if self._encode_new_garments(heads, device, dtype):
                continue                   # garments were dropped with their requests: take the heads again
            entries, failed = _prepare_photos_or_drop(heads, self.height, self.width, self.photo_filter)
            slots = iter(free)
            for i, entry in enumerate(entries):
                req = self.waiting.popleft()
                g = self._garment(req, device, dtype)       # a dropped request's garment stays known to later requests
                if i in failed:
                    self.failed[req.ticket] = failed[i]
                    self.stats["failed"] += 1
                    continue
                s = next(slots)
                seed = self._seed(req)
                gen = torch.Generator(device).manual_seed(seed) if seed is not None else None
                prep = self._prepare_request(req, gen) if entry is None else self._prepare_request(req, gen, entry)
                if self.mixed:             # the slot runs plan j; the garment's page is keyed by that plan's timesteps
                    j = self._plan_index[_preset_name(self, req)]
                    T, t_table = self.plans[j].T, self.plans[j].t_table[:self.plans[j].T]
                    key = (req.garment_id, tuple(float(t) for t in t_table))
                else:
                    j, T, t_table, key = None, self.T, None, req.garment_id
                page, host = (None, None) if self.garment_kv_bytes is None else self._pin_garment(key, g, t_table)
                self.den.admit(s, cloth_latents=g["latents"], image_embeds=g["image_embeds"],
                               text_embeds_cloth=g["text_embeds_cloth"], page=page,
                               **({} if host is None else dict(host_page=host)), **prep)
                self.slots[s] = dict(req=req, gen=gen, step=0, page=page, plan=j, T=T, photo=entry)
                if host is not None:
                    self.slots[s]["host_page"] = host
                self.stats["admitted"] += 1
            free = [s for s, e in enumerate(self.slots) if e is None]
        self._count_streamed()

    def _count_streamed(self):
        if self.garment_kv_host_bytes is not None and self.den is not None:
            rows, nbytes = self.den.take_streamed()
            self.stats["garment_rows_streamed"] += rows
            self.stats["garment_bytes_streamed"] += nbytes

    def _pin_garment(self, key, g, t_table=None):
        """Pool mode: (device page, None) or, with a host tier, (None, host page) holding `key`, pinned for one more
        slot. Lookup order: a device page; a host page (the slot streams from it and pins no device page, so P >= slots
        still holds for the device pages); then a miss (_pin_page)."""
        if self.garment_kv_host_bytes is not None and key not in self.page_of:
            q = self.host_page_of.get(key)
            if q is not None:
                self.host_page_of.move_to_end(key)
                self.host_pins[q] += 1
                self.stats["garment_host_hits"] += 1
                return None, q
        return self._pin_page(key, g, t_table), None

    def _pin_page(self, key, g, t_table=None):
        """Pool mode: the page holding `key` (the garment id; with the mixed-kind step, (garment id, the plan's
        timesteps t_table)), pinned for one more slot. A miss fills a free page, else the least recently admitted
        unpinned one (one exists: a free slot means at most slots - 1 pinned pages, and P >= slots), and with a host
        tier writes it through to a host page."""
        p = self.page_of.get(key)
        if p is not None:
            self.page_of.move_to_end(key)
            self.stats["garment_page_hits"] += 1
        else:
            if self.free_pages:
                p = self.free_pages.pop(0)
            else:
                victim = next(k for k, q in self.page_of.items() if self.pins[q] == 0)
                p = self.page_of.pop(victim)
                self.stats["garment_page_evictions"] += 1
            self.den.fill_page(p, g["latents"], g["text_embeds_cloth"], *(() if t_table is None else (t_table,)))
            self.page_of[key] = p
            self.stats["garment_page_fills"] += 1
            if self.garment_kv_host_bytes is not None:
                self._write_through(key, p)
        self.pins[p] += 1
        return p

    def _write_through(self, key, p):
        """Host tier: device page p, just filled with `key`, copied to a free host page, else to the least recently used
        unpinned one; skipped (and counted) when every host page is pinned. The device page is valid either way."""
        if self.free_host_pages:
            q = self.free_host_pages.pop(0)
        else:
            victim = next((k for k, q in self.host_page_of.items() if self.host_pins[q] == 0), None)
            if victim is None:
                self.stats["garment_host_skipped"] += 1
                return
            q = self.host_page_of.pop(victim)
            self.stats["garment_host_evictions"] += 1
        self.den.write_through(p, q)
        self.host_page_of[key] = q
        self.stats["garment_host_writes"] += 1

    def _decode(self, latents):
        if self.output_type == "latent":
            return latents
        return self.pipe._postprocess(self.pipe._decode_latents(latents), self.output_type)

    def _check_freeu(self):
        """The try-on UNet's FreeU setting is read at configure. A request must not run part of its steps with other
        values, so a change while requests run raises; a change while the server is idle re-configures. The garment
        UNet does not run FreeU, so garment latents, K/V and pool pages stay valid."""
        if not getattr(self, "_configured", False) or _freeu(self.pipe) == self._freeu:
            return
        if any(e is not None for e in self.slots):
            raise RuntimeError(f"the pipeline's FreeU setting changed to {_freeu(self.pipe)} while requests run with "
                               f"{self._freeu}: change it when the server is idle")
        self._configured = False

    @torch.no_grad()
    def step(self, use_graph=True):
        """Admits, runs one denoise step, decodes and frees the slots that finished. Returns {ticket: image}."""
        self._check_freeu()
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
            plan = den if e["plan"] is None else self.plans[e["plan"]]      # the draws of the slot's own run
            n = variance_noise(plan, e["step"], (1, 4, *self.latent_size), e["gen"], device, den.latents.dtype)
            if n is not None:
                noises[s] = n
        steps = [None if e is None else e["step"] if e["plan"] is None else (e["plan"], e["step"]) for e in self.slots]
        latents = den.step(steps, noises, use_graph=use_graph and getattr(self.pipe, "use_cuda_graph", True))
        self._count_streamed()
        self.stats["steps"] += 1
        self.stats["slot_steps"] += len(active)
        done = []
        for s in active:
            self.slots[s]["step"] += 1
            if self.slots[s]["step"] == self.slots[s]["T"]:
                done.append(s)
        if not done:
            self.last_latents = {}
            return {}
        final = latents[done].clone()
        tickets = [self.slots[s]["req"].ticket for s in done]
        self.last_latents = dict(zip(tickets, final))
        entries = [self.slots[s]["photo"] for s in done]
        if self.output_type != "latent" and any(e is not None for e in entries):
            # photo requests finishing at this step are pasted back in one launch
            images = _decode_with_photos(self.pipe, self.output_type, final, entries,
                                         [self.slots[s]["req"] for s in done])
        else:
            images = self._decode(final)
        for s in done:
            den.release(s)
            if self.slots[s]["page"] is not None:      # the page stays resident as a cache entry
                self.pins[self.slots[s]["page"]] -= 1
            if self.slots[s].get("host_page") is not None:
                self.host_pins[self.slots[s]["host_page"]] -= 1
            self.slots[s] = None
        self.stats["images"] += len(done)
        return {t: images[i] for i, t in enumerate(tickets)}

    def run(self, use_graph=True):
        """Steps until every submitted request is finished; returns {ticket: image}."""
        out = {}
        while self.pending():
            out.update(self.step(use_graph=use_graph))
        return out
