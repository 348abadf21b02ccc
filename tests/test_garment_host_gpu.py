"""The host tier of the garment K/V pool on the GPU, at the tiny config in the fp16 and fp8 formats:
  * a trace over more garments than device pages (P = S) gives every request the bits of a server whose device pool
    holds every garment, with host hits; at slots = 1 a streamed request gets TryOnServer(max_batch=1)'s bits;
  * a page evicted right after its fill leaves a host copy equal to the page it came from;
  * one step mixing device-page rows, ring rows and idle rows, with presets of different step counts: graph replay
    equals eager launches;
  * with the host tier off, the pool's shapes and the step's launches are those without the feature.
"""
import pytest
import torch

from test_continuous_gpu import _drive, _err, _pipe
from test_continuous_pool_gpu import _pool_server, _request, tiny_modules  # noqa: F401

pytestmark = pytest.mark.gpu
FORMATS = ["fp16", "fp8"]


def _server(tiny, fmt, pages, host_pages=None, slots=2, presets=None):
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.serving import ContinuousTryOnServer
    if presets is None:
        srv = _pool_server(tiny, 1, slots=slots)
    else:
        srv = ContinuousTryOnServer(_pipe(tiny), height=MG.H, width=MG.W, slots=slots, seed=7, output_type="pt",
                                    presets=presets, default_preset=next(iter(presets)), garment_kv_bytes=0)
    srv.pipe.set_garment_kv_precision(fmt)
    srv.garment_kv_bytes = pages * srv.page_bytes()
    if host_pages is not None:
        srv.garment_kv_host_bytes = host_pages * srv.page_bytes()
    return srv


@pytest.fixture
def restore_format(tiny_modules):  # noqa: F811
    yield
    tiny_modules["net_t"].set_garment_kv_precision("fp16")


def _script(tiny, garments):
    return [([_request(tiny, 40 + k, g)], 1) for k, g in enumerate(garments)]


@pytest.mark.parametrize("fmt", FORMATS)
def test_trace_over_more_garments_than_device_pages(tiny_modules, restore_format, fmt):  # noqa: F811
    garments = "ABCDABCADB"
    full = _server(tiny_modules, fmt, pages=4)
    _, want, _ = _drive(full, _script(tiny_modules, garments))
    srv = _server(tiny_modules, fmt, pages=2, host_pages=4)
    try:
        _, got, _ = _drive(srv, _script(tiny_modules, garments))
        st = dict(srv.stats)
        print("HOST_REPORT", fmt, {k: v for k, v in st.items() if k.startswith("garment")})
        assert full.stats["garment_page_fills"] == 4 and st["garment_host_hits"] >= 3
        assert st["garment_page_fills"] == st["garment_host_writes"] == 4 and st["garment_host_skipped"] == 0
        assert st["garment_rows_streamed"] == 4 * st["garment_host_hits"]         # every step of every host hit
        assert sorted(got) == sorted(want) == list(range(len(garments)))
        assert all(torch.equal(got[k], want[k]) for k in want), [_err(got[k], want[k]) for k in want]
        assert srv.den.host.blocks[0][0].is_pinned() if fmt == "fp8" else srv.den.host.blocks[0].is_pinned()
    finally:
        srv.close()
    assert srv.den is None


@pytest.mark.parametrize("fmt", FORMATS)
def test_streamed_single_slot_equals_batch_mode(tiny_modules, restore_format, fmt):  # noqa: F811
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.serving import TryOnServer
    reqs = lambda: [_request(tiny_modules, 50, "A"), _request(tiny_modules, 51, "B"),  # noqa: E731
                    _request(tiny_modules, 52, "A")]
    srv = _server(tiny_modules, fmt, pages=1, host_pages=2, slots=1)
    try:
        _, lat, _ = _drive(srv, [(reqs(), 0)])
        assert srv.stats["garment_host_hits"] == 1 and srv.stats["garment_page_fills"] == 2
    finally:
        srv.close()
    for k, r in enumerate(reqs()):
        pipe = _pipe(tiny_modules)
        pipe.set_garment_kv_precision(fmt)
        ref_srv = TryOnServer(pipe, height=MG.H, width=MG.W, num_inference_steps=4, guidance_scale=2.0, max_batch=1,
                              seed=r.seed, garment_cache_bytes=0, output_type="latent")
        ref_srv.submit(r)
        ref_srv.run()
        assert torch.equal(lat[k], pipe._last_latents[0]), (k, _err(lat[k], pipe._last_latents[0]))


@pytest.mark.parametrize("fmt", FORMATS)
def test_evicted_page_leaves_an_equal_host_copy(tiny_modules, restore_format, fmt):  # noqa: F811
    from idm_vton_b200.denoise import SlotDenoiser, kv_parts
    from idm_vton_b200.scheduler import DDPMScheduler
    from test_continuous_pool_gpu import _loop_inputs
    tiny_modules["net_t"].set_garment_kv_precision(fmt)
    eng_t, eng_g = tiny_modules["net_t"].engine(), tiny_modules["net_g"].engine()
    h, w, T = 20, 12, 5
    sch = DDPMScheduler()
    sch.set_timesteps(T)
    a, b = _loop_inputs(tiny_modules, h, w, 3), _loop_inputs(tiny_modules, h, w, 4)
    den = SlotDenoiser(eng_t, eng_g, 2, pages=2, host_pages=3)
    try:
        den.configure(sch, sch.timesteps, h, w)
        den.fill_page(1, a["cloth_latents"], a["text_embeds_cloth"])
        want = [[p[T:2 * T].clone() for p in kv_parts(kv)] for kv in den.pool]
        den.write_through(1, 2)
        den.fill_page(1, b["cloth_latents"], b["text_embeds_cloth"])     # evicts right away: waits for the copy
        torch.cuda.synchronize()
        for kv, host, ref in zip(den.pool, den.host.blocks, want):
            for part, hpart, r in zip(kv_parts(kv), kv_parts(host), ref):
                assert torch.equal(hpart[2 * T:3 * T], r.cpu())
        assert not torch.equal(kv_parts(den.pool[0])[0][T:2 * T].cpu(), kv_parts(den.host.blocks[0])[0][2 * T:])
    finally:
        den.release_host()


@pytest.mark.parametrize("fmt", FORMATS)
def test_mixed_rows_and_presets_graph_equals_eager(tiny_modules, restore_format, fmt):  # noqa: F811
    """Three slots, presets of 4 and 3 steps: in one step a slot reads a device page, another streams from the host
    and the third is idle or at another phase. Graph replay against eager launches, and against a server whose device
    pool holds every garment."""
    from test_presets_gpu import _preset

    def script():
        out = []
        for k, (g, name) in enumerate(zip("ABCDABCDAB", ["ddpm", "dpmpp"] * 5)):
            r = _request(tiny_modules, 60 + k, g)
            r.sampling = name
            out.append(([r], 1 + k % 2))
        return out
    presets = lambda: {"ddpm": _preset("ddpm"), "dpmpp": _preset("dpmpp")}  # noqa: E731
    mixed_steps = []
    runs = {}
    for name, use_graph, pages, host in (("graph", True, 3, 6), ("eager", False, 3, 6), ("full", True, 4, None)):
        srv = _server(tiny_modules, fmt, pages=pages, host_pages=host, slots=3, presets=presets())
        try:
            def record(srv=srv):
                return {"idle" if e is None else "host" if e.get("host_page") is not None else "device"
                        for e in srv.slots}
            out, lat = {}, {}
            for reqs, n in script():
                for r in reqs:
                    srv.submit(r)
                for _ in range(n):
                    srv._admit()
                    if host is not None and use_graph:
                        mixed_steps.append(record())
                    out.update(srv.step(use_graph=use_graph))
                    lat.update(srv.last_latents)
            while srv.pending():
                out.update(srv.step(use_graph=use_graph))
                lat.update(srv.last_latents)
            runs[name] = (lat, dict(srv.stats))
        finally:
            srv.close()
    assert any({"host", "device"} <= k for k in mixed_steps), mixed_steps
    assert runs["graph"][1]["garment_host_hits"] >= 2, runs["graph"][1]
    assert runs["graph"][1] == runs["eager"][1]
    for k, v in runs["full"][0].items():
        assert torch.equal(runs["graph"][0][k], v) and torch.equal(runs["eager"][0][k], v), k


def test_host_tier_off_keeps_the_pool_and_the_step(tiny_modules):  # noqa: F811
    from idm_vton_b200 import lib as L
    counts = {}
    for host in (None, 4):
        srv = _server(tiny_modules, "fp16", pages=2, host_pages=host, slots=2)
        try:
            srv.submit(_request(tiny_modules, 40, "A"))
            srv.step()
            T = srv.den.T_page
            rows = [p.shape[0] for p in srv.den.pool]
            assert rows == [2 * T + (0 if host is None else 4)] * len(rows)
            n0 = L.launch_count()
            srv.den.step([1, None], use_graph=False)
            counts[host] = L.launch_count() - n0
            if host is None:
                assert srv.den.host is None and srv.den._side is None
                assert not any(k.startswith("garment_host") for k in srv.stats)
            srv.run()
        finally:
            srv.close()
    assert counts[None] == counts[4] > 0, counts


def test_host_budget_refusal_before_any_launch(tiny_modules):  # noqa: F811
    from idm_vton_b200 import lib as L
    srv = _server(tiny_modules, "fp16", pages=2, slots=2)
    srv.garment_kv_host_bytes = srv.page_bytes() - 1
    srv.submit(_request(tiny_modules, 40, "A"))
    n0 = L.launch_count()
    with pytest.raises(ValueError, match=f"no garment K/V page of {srv.page_bytes()} bytes"):
        srv.step()
    assert L.launch_count() == n0
