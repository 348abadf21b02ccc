"""Pool mode of continuous batching without a GPU: the garment-page table of serving.ContinuousTryOnServer on a stand-in
denoiser (pin, share, unpin, least-recently-used eviction, fills and hits), the per-slot row table of
denoise.SlotDenoiser, the page size, the refusals, and the b200vton_attention_rows entry point (declared, exported,
argument checks)."""
import ctypes
import os
import random
import types

import pytest
import torch

from test_continuous_cpu import _cpu_pipe, _req, _schedulers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS_SYMBOLS = ("b200vton_cfg_ddpm_step_rows", "b200vton_cfg_solver_step_rows", "b200vton_nchw_to_nhwc_scaled_rows",
                "b200vton_attention_rows")


# ------------------------------------------------------------------------------------------------------------------
# the page table
# ------------------------------------------------------------------------------------------------------------------
class _FakePoolDen:
    """Stand-in SlotDenoiser in pool mode: page p holds the garment last filled into it; latents[s] counts steps."""

    def __init__(self, S, T, P):
        self.S, self.T, self.P = S, T, P
        self.latents = torch.zeros(S, 4, 2, 2)
        self.step_draws, self.noise_applied = [False] * T, True
        self.content = [None] * P
        self.page = [None] * S
        self.log = []

    def fill_page(self, p, cloth_latents, text_embeds_cloth):
        self.log.append(("fill", p, cloth_latents))
        self.content[p] = cloth_latents

    def admit(self, s, page=None, **kw):
        self.log.append(("admit", s, page))
        self.page[s] = page

    def step(self, steps, noises=None, use_graph=True):
        for s, i in enumerate(steps):
            if i is not None:
                self.latents[s] += 1
        return self.latents

    def release(self, s):
        self.page[s] = None


def _pool_fake_server(S=2, T=3, P=2):
    from idm_vton_b200.serving import ContinuousTryOnServer

    class Srv(ContinuousTryOnServer):
        def _configure(self):
            self.den, self.T, self._configured = _FakePoolDen(S, T, P), T, True
            self._reset_pages(P)

        def _garment(self, req, device, dtype):
            self.garments[req.garment_id] = dict(latents=req.garment_id, image_embeds=None, text_embeds_cloth=None)
            return self.garments[req.garment_id]

        def _prepare_request(self, req, gen):
            return dict(latents=torch.tensor(float(req.ticket)))

        def _decode(self, latents):
            return latents

    pipe = types.SimpleNamespace(vae_scale_factor=8, _execution_device=torch.device("cpu"),
                                 unet=types.SimpleNamespace(dtype=torch.float32))
    return Srv(pipe, height=32, width=32, slots=S, num_inference_steps=T, seed=1, garment_kv_bytes=1)


def _check_invariants(srv):
    den = srv.den
    held = [e["page"] for e in srv.slots if e is not None]
    assert den.page == [None if e is None else e["page"] for e in srv.slots]
    for s, e in enumerate(srv.slots):                      # every slot reads its own garment's page
        if e is not None:
            assert den.content[e["page"]] == e["req"].garment_id and srv.page_of[e["req"].garment_id] == e["page"]
    assert {p: n for p, n in srv.pins.items() if n} == {p: held.count(p) for p in set(held)}
    assert sorted(list(srv.page_of.values()) + srv.free_pages) == list(range(den.P))


def test_pages_are_pinned_shared_unpinned_and_kept():
    srv = _pool_fake_server(S=2, T=3, P=2)
    srv.submit(_req("A"))
    srv.submit(_req("A", cloth=False))
    srv.step()                                             # both slots read one page: one fill, one hit
    assert [e[0] for e in srv.den.log] == ["fill", "admit", "admit"] and srv.den.page == [0, 0]
    assert srv.stats["garment_page_fills"] == 1 and srv.stats["garment_page_hits"] == 1 and srv.pins[0] == 2
    _check_invariants(srv)
    srv.run()
    assert srv.pins[0] == 0 and srv.page_of == {"A": 0}   # unpinned, still resident
    srv.den.log.clear()
    srv.submit(_req("A", cloth=False))
    srv.step()                                             # a later request for the garment: no fill
    assert srv.den.log == [("admit", 0, 0)] and srv.stats["garment_page_hits"] == 2
    _check_invariants(srv)


def test_miss_evicts_the_least_recently_used_unpinned_page():
    srv = _pool_fake_server(S=2, T=2, P=3)
    for g in "ABC":                                        # A, B in slots; C waits
        srv.submit(_req(g))
    srv.run()
    assert list(srv.page_of) == ["A", "B", "C"] and srv.free_pages == []
    srv.submit(_req("A", cloth=False))                     # hit: A becomes the most recent
    srv.step()
    srv.submit(_req("D"))                                  # miss: B is the least recently used unpinned page
    srv.step()
    assert "B" not in srv.page_of and srv.page_of["D"] == 1 and srv.stats["garment_page_evictions"] == 1
    _check_invariants(srv)
    srv.submit(_req("E"))                                  # A has finished; C is the least recently used, D is pinned
    srv.run()
    assert "C" not in srv.page_of and set(srv.page_of) == {"A", "D", "E"}
    assert srv.stats["garment_page_fills"] == 5 and srv.stats["garment_page_hits"] == 1


def test_a_free_page_always_exists_at_the_minimum_budget():
    """P = slots, many garments, random arrivals: every admission finds a page, no pinned page is ever refilled."""
    rnd = random.Random(3)
    srv = _pool_fake_server(S=3, T=4, P=3)
    n = 0
    for _ in range(60):
        for _ in range(rnd.randint(0, 2)):
            g = rnd.choice("ABCDEFG")
            srv.submit(_req(g))
            n += 1
        srv.step()
        if srv.den is not None:                            # configured at the first admission
            _check_invariants(srv)
    srv.run()
    assert srv.stats["images"] == n == srv.stats["admitted"]
    assert srv.stats["garment_page_fills"] + srv.stats["garment_page_hits"] == n


# ------------------------------------------------------------------------------------------------------------------
# the slot denoiser's row table and the page size
# ------------------------------------------------------------------------------------------------------------------
class _Blk:
    def __init__(self, c):
        self.c = c


def _engine(symbols=ROWS_SYMBOLS):
    L = types.SimpleNamespace(has_symbol=lambda n: n in symbols)
    return types.SimpleNamespace(L=L, device=torch.device("cpu"), ch=(8, 16),
                                 blocks=lambda: [_Blk(16), _Blk(16), _Blk(8)])


def test_page_size_from_the_shapes():
    from idm_vton_b200.denoise import garment_kv_bytes_per_step, garment_tokens
    eng = _engine()
    assert garment_tokens(eng, 5, 3) == [3 * 2, 3 * 2, 5 * 3]   # level 1 rounds up: (5-1)//2+1 x (3-1)//2+1
    assert garment_kv_bytes_per_step(eng, 5, 3) == 2 * (6 * 32 * 2) + 15 * 16 * 2
    # SDXL at 768x1024: 10 blocks of 640 channels over 3072 garment tokens, 60 of 1280 over 768
    sdxl = types.SimpleNamespace(ch=(320, 640, 1280), blocks=lambda: [_Blk(640)] * 10 + [_Blk(1280)] * 60)
    assert 30 * garment_kv_bytes_per_step(sdxl, 128, 96) == 9_437_184_000


def test_row_table_per_slot_and_its_checks():
    from idm_vton_b200.denoise import SlotDenoiser
    from idm_vton_b200.scheduler import DDPMScheduler
    sch = DDPMScheduler()
    sch.set_timesteps(5)
    with pytest.raises(ValueError, match="one garment K/V page per slot"):
        SlotDenoiser(_engine(), _engine(), 3, pages=2)
    den = SlotDenoiser(_engine(), _engine(), 3, pages=4)
    den.configure(sch, sch.timesteps, 4, 4)
    assert den.x_g is None and den.t_g is None and den.rows.tolist() == [-1, -1, -1]
    assert [tuple(p.shape) for p in den.pool] == [(20, 4, 32), (20, 4, 32), (20, 16, 16)]
    den.page = [3, None, 0]
    den.gather([4, None, 2])
    assert den.rows.tolist() == [3 * 5 + 4, -1, 2] and den.rows.dtype == torch.int32
    with pytest.raises(ValueError, match="holds no garment K/V page"):
        den.gather([4, 1, 2])
    den.page = [4, None, 0]                                # a page outside the pool
    with pytest.raises(ValueError, match=r"outside \[-1, 20\)"):
        den.gather([0, None, 0])
    with pytest.raises(ValueError, match=r"outside \[0, 4\)"):
        den.fill_page(4, torch.zeros(1, 4, 4, 4), torch.zeros(1, 77, 8))


def test_pool_refusals():
    from idm_vton_b200 import lib
    from idm_vton_b200.denoise import SlotDenoiser
    from idm_vton_b200.scheduler import DDPMScheduler
    from idm_vton_b200.serving import ContinuousTryOnServer
    sch = DDPMScheduler()
    sch.set_timesteps(4)
    with pytest.raises(NotImplementedError, match="b200vton_attention_rows"):
        SlotDenoiser(_engine(ROWS_SYMBOLS[:3]), _engine(), 2, pages=2).configure(sch, sch.timesteps, 4, 4)
    SlotDenoiser(_engine(ROWS_SYMBOLS[:3]), _engine(), 2).configure(sch, sch.timesteps, 4, 4)   # default mode: not needed
    # a budget below one page per slot, refused at the first step before anything runs
    pipe, _, _ = _cpu_pipe(_schedulers()["ddpm"][0])
    pipe.unet.engine = _engine
    assert pipe.vae_scale_factor == 2
    page = 3 * (2 * (8 * 8 * 32 * 2) + 16 * 16 * 16 * 2)   # 3 steps at 16x16 latents (32x32 pixels)
    lib.load()
    n0 = lib.launch_count()
    for budget, ok in ((2 * page - 1, False), (2 * page, True)):
        srv = ContinuousTryOnServer(pipe, height=32, width=32, slots=2, num_inference_steps=3, garment_kv_bytes=budget)
        assert srv.page_bytes() == page
        if ok:
            assert srv._pages(3) == 2
            continue
        srv.submit(_req("A"))
        with pytest.raises(ValueError, match=f"holds 1 garment K/V pages of {page} bytes"):
            srv.step()
    assert lib.launch_count() == n0


# ------------------------------------------------------------------------------------------------------------------
# the C ABI
# ------------------------------------------------------------------------------------------------------------------
def test_attention_rows_declared_exported_and_validated():
    from test_fp8_cpu import _declared_args
    from idm_vton_b200 import build, lib
    name = "b200vton_attention_rows"
    header = open(os.path.join(ROOT, "include", "b200vton.h")).read()
    so = ctypes.CDLL(build.build())
    assert hasattr(so, name) and lib.OPTIONAL_SIGNATURES[name] == _declared_args(header, name)
    raw = lib.load()
    assert lib.has_symbol(name)
    fn = getattr(raw, name)
    n0 = lib.launch_count()

    def call(rows=256, n1=4, b1=2, k1=64, off=0, B=2):
        return fn(64, 128, 64, 64, 128, k1, 64, 128, 64, 128, B, 2, 4, 4, n1, b1, off, rows, 0.125, 0, None)
    assert call(rows=None) == 1 and b"kv1_rows is null" in raw.b200vton_last_error()
    assert call(rows=258) == 1 and b"aligned" in raw.b200vton_last_error()
    for kw in (dict(n1=0), dict(b1=0), dict(k1=None)):
        assert call(**kw) == 1 and b"segment-1" in raw.b200vton_last_error(), kw
    for off in (-1, 2):
        assert call(off=off) == 1 and b"kv1_off" in raw.b200vton_last_error()
    assert lib.launch_count() == n0


def test_library_without_attention_rows_refuses_in_the_binding():
    from idm_vton_b200 import lib
    lib.load()
    present = set(lib._present)
    try:
        lib._present.discard("b200vton_attention_rows")
        with pytest.raises(NotImplementedError, match="b200vton_attention_rows"):
            lib.attention_rows(None, None, None, None, None, None)
    finally:
        lib._present.update(present)
