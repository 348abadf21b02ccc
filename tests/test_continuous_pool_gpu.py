"""Continuous batching with a pool of hoisted garment K/V pages, on the GPU:
  * b200vton_attention_rows: a row table over a pool against b200vton_attention on the K/V gathered by the same table,
    with and without CFG rows, Ng off a tile multiple and a row at P*T - 1; a -1 entry against the zero-K/V closed
    form; and against float64, where the table-ignored mutant must lie >= 4x further away than the kernel;
  * SlotDenoiser.fill_page: a page holds TryOnDenoiser's gkv_all of the same garment alone, in any page;
  * ContinuousTryOnServer(garment_kv_bytes=...) at the tiny config: invariance of a request's latents to its
    neighbours, slot, order, page misses / hits and page sharing; graph replay against eager launches across fills and
    evictions; a hit runs no garment pass; slots = 1 against TryOnServer(max_batch=1); the refusals;
  * 2 slots at SDXL width against the batch-mode denoiser, gated as test_continuous_gpu.py gates the default mode.
"""
import pytest
import torch

from test_attention_pipeline_gpu import TOL_ATTN, head_ref, rel_err, rnd16
from test_continuous_gpu import _bound, _drive, _err, _pair_inputs, _pipe, _report

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------
# kernel
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [True, False])
def test_attention_rows_against_gathered_kv_and_float64(cfg):
    from idm_vton_b200 import lib as L
    S, H, Nq, N0, N1, P, T = 3, 2, 200, 257, 200, 4, 5       # N1 off a multiple of 128
    C = H * 64
    off = S if cfg else 0
    B = off + S
    q, k0, v0 = (rnd16(B, n, C, seed=700 + i, device="cuda") for i, n in enumerate((Nq, N0, N0)))
    pool = rnd16(P * T, N1, 2 * C, seed=710, device="cuda")
    table = [P * T - 1, 7, 0]                                 # the last row of the last page; no row equals its sample
    rows = torch.tensor(table, dtype=torch.int32, device="cuda")
    out = L.attention_rows(q, k0, v0, pool[..., :C], pool[..., C:], rows, kv1_off=off, heads=H)
    g = pool[rows.long()].contiguous()
    ref = L.attention(q, k0, v0, g[..., :C], g[..., C:], kv1_off=off, heads=H)
    assert torch.equal(out, ref)
    errs, mut = [], []
    for b in range(B):
        for h in range(H):
            c, cv = slice(64 * h, 64 * h + 64), slice(C + 64 * h, C + 64 * h + 64)
            if b < off:
                truth = head_ref(q[b, :, c], k0[b, :, c], v0[b, :, c], n_zero=N1)
                mutant = truth
            else:
                r, m = table[b - off], b - off                # the mutant ignores the table: row = sample index
                truth = head_ref(q[b, :, c], torch.cat([k0[b, :, c], pool[r, :, c]]), torch.cat([v0[b, :, c], pool[r, :, cv]]))
                mutant = head_ref(q[b, :, c], torch.cat([k0[b, :, c], pool[m, :, c]]), torch.cat([v0[b, :, c], pool[m, :, cv]]))
                mut.append(rel_err(mutant, truth))
            errs.append(rel_err(out[b, :, c], truth))
    _report(case=f"attention_rows cfg={cfg}", err=max(errs), mutant=min(mut))
    assert max(errs) <= TOL_ATTN and max(errs) <= 0.25 * min(mut), (max(errs), min(mut))
    # -1 entries: the zero-K/V closed form of the existing entry point, bit for bit, and the other samples unchanged
    idle = torch.tensor([-1, 7, -1], dtype=torch.int32, device="cuda")
    out_i = L.attention_rows(q, k0, v0, pool[..., :C], pool[..., C:], idle, kv1_off=off, heads=H)
    zero = L.attention(q, k0, v0, n1=N1, kv1_off=B, heads=H)         # every sample: N1 zero K/V tokens, closed form
    for j, r in enumerate(idle.tolist()):
        assert torch.equal(out_i[off + j], zero[off + j] if r < 0 else out[off + j]), j
    assert torch.equal(out_i[:off], out[:off])


# ------------------------------------------------------------------------------------------------
# pages
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny_modules():
    from oracle import unet_ref as R
    from idm_vton_b200 import unet as U
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t, sd_g = R.make_state_dict(cfg_t, seed=11), R.make_state_dict(cfg_g, seed=22)
    net_t = U.UNet2DConditionModel(cfg_t, sd_t).to("cuda", torch.float16)
    net_g = U.UNet2DConditionModelGarment(cfg_g, sd_g).to("cuda", torch.float16)
    return dict(cfg_t=cfg_t, cfg_g=cfg_g, net_t=net_t, net_g=net_g)


def _loop_inputs(tiny, h, w, seed):
    from test_fullsize_gpu import _forward_inputs
    return _forward_inputs(tiny["cfg_t"], tiny["cfg_g"], 1, h, w, seed=seed)


def test_filled_page_equals_batch_mode_gkv_in_any_page(tiny_modules):
    from idm_vton_b200.denoise import SlotDenoiser, TryOnDenoiser
    from idm_vton_b200.scheduler import DDPMScheduler
    eng_t, eng_g = tiny_modules["net_t"].engine(), tiny_modules["net_g"].engine()
    h, w, T = 20, 12, 5
    sch = DDPMScheduler()
    sch.set_timesteps(T)
    inp, other = _loop_inputs(tiny_modules, h, w, 3), _loop_inputs(tiny_modules, h, w, 4)
    den = TryOnDenoiser(eng_t, eng_g)
    den.prepare(**inp, guidance_scale=2.0)
    den.set_step_tables(sch, sch.timesteps)
    assert den.window == T
    want = [g.clone() for g in den.gkv_all]
    slot = SlotDenoiser(eng_t, eng_g, 2, pages=3)
    slot.configure(sch, sch.timesteps, h, w)
    slot.fill_page(2, other["cloth_latents"], other["text_embeds_cloth"])
    for p in (1, 0):
        slot.fill_page(p, inp["cloth_latents"], inp["text_embeds_cloth"])
        assert all(torch.equal(pool[p * T:(p + 1) * T], g) for pool, g in zip(slot.pool, want)), p
    assert not torch.equal(slot.pool[0][2 * T:], want[0])     # another garment's page holds other values


# ------------------------------------------------------------------------------------------------
# the server (tiny config)
# ------------------------------------------------------------------------------------------------
GARMENT_SEEDS = {"A": 1001, "B": 1002, "C": 1003, "D": 1004}


def _request(tiny, person_seed, garment, seed=7):
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.serving import TryOnRequest
    i = MG.make_call_inputs(tiny["cfg_t"], B=1, seed=person_seed)
    gi = MG.make_call_inputs(tiny["cfg_t"], B=1, seed=GARMENT_SEEDS[garment])
    return TryOnRequest(garment_id=garment, image=i["image"][0].cuda(), mask_image=i["mask_image"][0].cuda(),
                        pose_img=i["pose_img"][0], prompt_embeds=i["prompt_embeds"][0],
                        negative_prompt_embeds=i["negative_prompt_embeds"][0],
                        pooled_prompt_embeds=i["pooled_prompt_embeds"][0],
                        negative_pooled_prompt_embeds=i["negative_pooled_prompt_embeds"][0], cloth=gi["cloth"][0],
                        ip_adapter_image=gi["ip_adapter_image"][0], text_embeds_cloth=gi["text_embeds_cloth"][0],
                        seed=seed)


def _pool_server(tiny, pages, kind="ddpm", slots=3, steps=4, output_type="pt"):
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.serving import ContinuousTryOnServer
    srv = ContinuousTryOnServer(_pipe(tiny, kind), height=MG.H, width=MG.W, slots=slots, num_inference_steps=steps,
                                guidance_scale=2.0, seed=7, output_type=output_type, garment_kv_bytes=0)
    srv.garment_kv_bytes = pages * srv.page_bytes()
    return srv


def test_pool_request_result_is_independent_of_neighbours_pages_and_order(tiny_modules):
    """A request's final latents are the same bits alone (page miss), beside requests at other phases in another slot,
    at another arrival order, on a page hit after its garment's page was filled by an earlier request, and sharing its
    page with a request of the same garment at another phase."""
    t = lambda: _request(tiny_modules, 40, "A")  # noqa: E731
    x = lambda: _request(tiny_modules, 41, "B")  # noqa: E731
    y = lambda: _request(tiny_modules, 42, "C")  # noqa: E731
    same = lambda: _request(tiny_modules, 43, "A")  # noqa: E731
    _, lat_a, slot_a = _drive(_pool_server(tiny_modules, 3), [([t()], 0)])
    _, lat_b, slot_b = _drive(_pool_server(tiny_modules, 3), [([x()], 2), ([y()], 1), ([t()], 0)])
    _, lat_c, slot_c = _drive(_pool_server(tiny_modules, 4), [([y()], 1), ([t()], 1), ([x()], 0)])
    srv_d = _pool_server(tiny_modules, 3)
    _, lat_d, _ = _drive(srv_d, [([same()], 5), ([x()], 1), ([t()], 0)])         # hit on a resident page
    srv_e = _pool_server(tiny_modules, 3)
    _, lat_e, slot_e = _drive(srv_e, [([same()], 2), ([x()], 0), ([t()], 0)])     # shares the page at another phase
    assert slot_a[0] == 0 and slot_b[2] == 2 and slot_c[1] == 1 and slot_e[2] == 2
    assert srv_d.stats["garment_page_hits"] == 1 and srv_d.stats["garment_page_fills"] == 2
    assert srv_e.stats["garment_page_hits"] == 1 and srv_e.stats["garment_page_fills"] == 2
    for name, lat, k in (("neighbours", lat_b, 2), ("order", lat_c, 1), ("hit", lat_d, 2), ("shared", lat_e, 2)):
        assert torch.equal(lat[k], lat_a[0]), name
    assert not torch.equal(lat_e[0], lat_a[0])                    # the page's other reader is another person


def test_pool_graph_replay_equals_eager_over_fills_and_evictions(tiny_modules):
    script = lambda: [([_request(tiny_modules, 41, "B")], 2), ([_request(tiny_modules, 42, "C")], 1),  # noqa: E731
                      ([_request(tiny_modules, 40, "A"), _request(tiny_modules, 43, "D")], 3),
                      ([_request(tiny_modules, 44, "B"), _request(tiny_modules, 45, "A")], 0)]
    for kind in ("ddpm", "dpmpp"):
        srv_g, srv_e = _pool_server(tiny_modules, 2, kind, slots=2), _pool_server(tiny_modules, 2, kind, slots=2)
        img_g, lat_g, _ = _drive(srv_g, script(), use_graph=True)
        img_e, lat_e, _ = _drive(srv_e, script(), use_graph=False)
        assert sorted(lat_g) == sorted(lat_e) == list(range(6))
        assert all(torch.equal(lat_g[k], lat_e[k]) and torch.equal(img_g[k], img_e[k]) for k in lat_g), kind
        assert srv_g.stats == srv_e.stats and srv_g.stats["garment_page_evictions"] >= 2, srv_g.stats


def test_page_hit_runs_no_garment_pass(tiny_modules, monkeypatch):
    """Admission launches on a hit are those of a miss (garment already encoded) minus one page fill, and the garment
    UNet is not called."""
    from idm_vton_b200 import lib as L
    srv = _pool_server(tiny_modules, 2, slots=2)
    _drive(srv, [([_request(tiny_modules, 40, "A"), _request(tiny_modules, 41, "B")], 0)])
    _drive(srv, [([_request(tiny_modules, 42, "C")], 0)])           # evicts A's page (least recently used)
    assert "A" not in srv.page_of and srv.stats["garment_page_evictions"] == 1
    calls = []
    real = type(srv.den.garment).forward
    monkeypatch.setattr(type(srv.den.garment), "forward", lambda self, *a, **k: calls.append(1) or real(self, *a, **k))

    def admit(req):
        srv.submit(req)
        n0, c0 = L.launch_count(), len(calls)
        srv._admit()
        return L.launch_count() - n0, len(calls) - c0
    miss, miss_calls = admit(_request(tiny_modules, 43, "A"))      # A is encoded; its page must be filled again
    hit, hit_calls = admit(_request(tiny_modules, 44, "A"))        # shares the page just filled
    n0 = L.launch_count()
    srv.den.fill_page(1 - srv.page_of["A"], srv.garments["A"]["latents"], srv.garments["A"]["text_embeds_cloth"])
    fill = L.launch_count() - n0
    _report(case="hit launches", miss=miss, hit=hit, fill=fill)
    assert miss_calls > 0 and hit_calls == 0 and miss - hit == fill > 0, (miss, hit, fill)


def test_pool_single_slot_equals_batch_mode(tiny_modules):
    """At slots = 1 the pool server runs the launches of TryOnServer(max_batch=1): the garment passes of one garment at
    TryOnDenoiser's chunking, the try-on UNet at batch 2 reading the same K/V rows. The final latents are the same bits."""
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.serving import TryOnServer
    reqs = lambda: [_request(tiny_modules, 50, "A"), _request(tiny_modules, 51, "B"),  # noqa: E731
                    _request(tiny_modules, 52, "A")]
    _, lat, _ = _drive(_pool_server(tiny_modules, 1, slots=1), [(reqs(), 0)])
    exact, errs = [], []
    for k, r in enumerate(reqs()):
        pipe = _pipe(tiny_modules)
        srv = TryOnServer(pipe, height=MG.H, width=MG.W, num_inference_steps=4, guidance_scale=2.0, max_batch=1,
                          seed=r.seed, garment_cache_bytes=0, output_type="latent")
        srv.submit(r)
        srv.run()
        ref = pipe._last_latents[0]                                 # [1,4,h,w]: the batch of one
        exact.append(lat[k].dtype == ref.dtype and bool(torch.equal(lat[k], ref)))
        errs.append(_err(lat[k], ref))
    _report(case="pool slots=1 vs TryOnServer(max_batch=1)", bit_identical=exact, errs=errs)
    assert all(exact), errs


def test_pool_refusals_before_any_launch(tiny_modules, monkeypatch):
    from idm_vton_b200 import lib as L
    srv = _pool_server(tiny_modules, 2, slots=3)                   # 2 pages for 3 slots
    srv.submit(_request(tiny_modules, 40, "A"))
    n0 = L.launch_count()
    with pytest.raises(ValueError, match="pages of"):
        srv.step()
    assert L.launch_count() == n0
    srv = _pool_server(tiny_modules, 3, slots=3)
    srv.submit(_request(tiny_modules, 40, "A"))
    monkeypatch.setattr(L, "_present", L._present - {"b200vton_attention_rows"})
    with pytest.raises(NotImplementedError, match="b200vton_attention_rows"):
        srv.step()
    assert L.launch_count() == n0


# ------------------------------------------------------------------------------------------------
# SDXL width
# ------------------------------------------------------------------------------------------------
def test_fullsize_pool_slots_against_batch_mode():
    """SDXL-width UNets (random weights), 2 slots in pool mode, 3 DDPM steps, as test_fullsize_slots_against_batch_mode
    runs the default mode: request 0 alone for one step, request 1 joins at its step 0; gated on the batch-mode
    denoiser's own difference between running the two requests alone and together."""
    from test_fullsize_gpu import _forward_inputs
    from idm_vton_b200 import unet as U
    from idm_vton_b200.denoise import SlotDenoiser, TryOnDenoiser
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON, UNetEngine
    from idm_vton_b200.scheduler import DDPMScheduler
    eng_t = UNetEngine(SDXL_TRYON, U.random_state_dict(SDXL_TRYON, seed=11, device="cuda"), "tryon")
    eng_g = UNetEngine(SDXL_GARMENT, U.random_state_dict(SDXL_GARMENT, seed=22, device="cuda"), "garment")
    h, w, steps = 128, 96, 3
    sch = DDPMScheduler()
    sch.set_timesteps(30)
    ts = sch.timesteps[:steps]
    inps = [_forward_inputs(SDXL_TRYON, SDXL_GARMENT, 1, h, w, seed=s) for s in (3, 4)]
    g = torch.Generator(device="cuda").manual_seed(5)
    noises = [[torch.randn(1, 4, h, w, generator=g, device="cuda").half() for _ in range(steps)] for _ in inps]

    def batch_mode(inp, nz):
        den = TryOnDenoiser(eng_t, eng_g)
        den.prepare(**inp, guidance_scale=2.0)
        den.set_step_tables(sch, ts)
        for i in range(steps):
            den.step(i, nz[i])
        return den.latents.clone()

    refs = [batch_mode(inp, nz) for inp, nz in zip(inps, noises)]
    pair = batch_mode(_pair_inputs(inps[0], inps[1]), [torch.cat([noises[0][i], noises[1][i]]) for i in range(steps)])
    spread = max(_err(pair[0:1], refs[0]), _err(pair[1:2], refs[1]))
    torch.cuda.empty_cache()
    den = SlotDenoiser(eng_t, eng_g, 2, pages=2)
    den.configure(sch, ts, h, w, guidance_scale=2.0)

    def admit(s, inp):
        den.fill_page(s, inp["cloth_latents"], inp["text_embeds_cloth"])
        den.admit(s, latents=inp["latents"], mask=inp["mask"], masked_image_latents=inp["masked_image_latents"],
                  pose_latents=inp["pose_latents"], cloth_latents=inp["cloth_latents"], prompt_embeds=inp["prompt_embeds"],
                  add_text_embeds=inp["add_text_embeds"], add_time_ids=inp["add_time_ids"],
                  image_embeds=inp["image_embeds"], text_embeds_cloth=inp["text_embeds_cloth"], page=s)
    admit(0, inps[0])
    den.step([0, None], {0: noises[0][0]})
    admit(1, inps[1])
    den.step([1, 0], {0: noises[0][1], 1: noises[1][0]})
    den.step([2, 1], {0: noises[0][2], 1: noises[1][1]})
    out0 = den.latents[0:1].clone()
    den.step([None, 2], {1: noises[1][2]})
    out1 = den.latents[1:2].clone()
    errs = [_err(out0, refs[0]), _err(out1, refs[1])]
    mutant = _err(out0, refs[1])
    bound = _bound(spread)
    _report(case="fullsize pool S=2 3 steps", errs=errs, bit_identical=[bool(torch.equal(out0, refs[0])),
                                                                        bool(torch.equal(out1, refs[1]))],
            batch2_vs_batch1=spread, bound=bound, other_request=mutant)
    assert max(errs) <= bound and mutant >= 10 * bound, (errs, bound, mutant)
