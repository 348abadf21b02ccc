"""The host tier of the garment K/V pool without a GPU: the two-tier lookup of serving.ContinuousTryOnServer on a
stand-in denoiser that records its calls (lookup order, LRU per tier, host pins, write-through and its skips, the stats),
the budgets and refusals, and on denoise.SlotDenoiser with a stand-in engine and recorded CUDA streams and events: the
ring-row arithmetic, the rows the ring receives, and the event order of fills, write-throughs and streamed rows."""
import contextlib
import types

import pytest
import torch

from test_continuous_cpu import _cpu_pipe, _req, _schedulers
from test_continuous_pool_cpu import ROWS_SYMBOLS, _Blk


# ------------------------------------------------------------------------------------------------------------------
# the two tiers on a stand-in denoiser
# ------------------------------------------------------------------------------------------------------------------
class _FakeHostDen:
    """Stand-in SlotDenoiser with a host tier: device page p / host page q hold the garment last written into them."""

    def __init__(self, S, T, P, Q):
        self.S, self.T, self.P, self.Q = S, T, P, Q
        self.latents = torch.zeros(S, 4, 2, 2)
        self.step_draws, self.noise_applied = [False] * T, True
        self.content, self.host = [None] * P, [None] * Q
        self.page, self.host_page = [None] * S, [None] * S
        self.log = []
        self.rows = 0
        self.released = 0

    def fill_page(self, p, cloth_latents, text_embeds_cloth):
        self.log.append(("fill", p, cloth_latents))
        self.content[p] = cloth_latents

    def write_through(self, p, q):
        self.log.append(("write", p, q))
        self.host[q] = self.content[p]

    def admit(self, s, page=None, host_page=None, **kw):
        self.log.append(("admit", s, page, host_page))
        self.page[s], self.host_page[s] = page, host_page
        self.rows += host_page is not None          # the first row

    def step(self, steps, noises=None, use_graph=True):
        for s, i in enumerate(steps):
            if i is not None:
                self.latents[s] += 1
                self.rows += self.host_page[s] is not None and i + 1 < self.T
        return self.latents

    def take_streamed(self):
        out, self.rows = (self.rows, 10 * self.rows), 0
        return out

    def release(self, s):
        self.page[s] = self.host_page[s] = None

    def release_host(self):
        self.released += 1


def _host_server(S=2, T=3, P=2, Q=2):
    from idm_vton_b200.serving import ContinuousTryOnServer

    class Srv(ContinuousTryOnServer):
        def _configure(self):
            self.den, self.T, self._configured = _FakeHostDen(S, T, P, Q), T, True
            self._reset_pages(P, Q)

        def _garment(self, req, device, dtype):
            self.garments[req.garment_id] = dict(latents=req.garment_id, image_embeds=None, text_embeds_cloth=None)
            return self.garments[req.garment_id]

        def _prepare_request(self, req, gen):
            return dict(latents=torch.tensor(float(req.ticket)))

        def _decode(self, latents):
            return latents

    pipe = types.SimpleNamespace(vae_scale_factor=8, _execution_device=torch.device("cpu"),
                                 unet=types.SimpleNamespace(dtype=torch.float32))
    return Srv(pipe, height=32, width=32, slots=S, num_inference_steps=T, seed=1, garment_kv_bytes=1,
               garment_kv_host_bytes=1)


def _check(srv):
    den = srv.den
    for s, e in enumerate(srv.slots):
        if e is None:
            assert den.page[s] is None and den.host_page[s] is None
            continue
        g, q = e["req"].garment_id, e.get("host_page")
        if q is None:                                        # a device page of its garment
            assert den.page[s] == e["page"] == srv.page_of[g] and den.content[e["page"]] == g and den.host_page[s] is None
        else:                                                # a host page of its garment, and no device page
            assert den.host_page[s] == q == srv.host_page_of[g] and den.host[q] == g and e["page"] is None
    held = [e["page"] for e in srv.slots if e is not None and e["page"] is not None]
    streaming = [e["host_page"] for e in srv.slots if e is not None and e.get("host_page") is not None]
    assert {p: n for p, n in srv.pins.items() if n} == {p: held.count(p) for p in set(held)}
    assert {q: n for q, n in srv.host_pins.items() if n} == {q: streaming.count(q) for q in set(streaming)}
    assert sorted(list(srv.page_of.values()) + srv.free_pages) == list(range(den.P))
    assert sorted(list(srv.host_page_of.values()) + srv.free_host_pages) == list(range(den.Q))
    for g, q in srv.host_page_of.items():
        assert den.host[q] == g


def _kinds(log):
    return [e[0] for e in log]


def test_lookup_order_device_then_host_then_miss():
    srv = _host_server(S=2, T=2, P=2, Q=3)
    srv.submit(_req("A"))
    srv.submit(_req("B"))
    srv.step()                                               # two misses: fill, write-through, admit
    assert _kinds(srv.den.log) == ["fill", "write", "admit", "fill", "write", "admit"]
    assert srv.stats["garment_host_writes"] == 2 and srv.den.host[:2] == ["A", "B"]
    srv.run()
    srv.submit(_req("C"))                                    # a miss evicts A's device page; A stays on the host
    srv.run()
    assert "A" not in srv.page_of and srv.host_page_of["A"] == 0
    srv.den.log.clear()
    srv.submit(_req("B", cloth=False))                       # B: on the device and on the host -> the device page
    srv.submit(_req("A", cloth=False))                       # A: on the host only -> streams, no fill
    srv.step()
    assert srv.den.log == [("admit", 0, srv.page_of["B"], None), ("admit", 1, None, 0)]
    assert srv.stats["garment_page_hits"] == 1 and srv.stats["garment_host_hits"] == 1
    assert srv.stats["garment_page_fills"] == 3 and srv.host_pins[0] == 1
    _check(srv)
    srv.run()
    assert srv.host_pins[0] == 0 and "A" not in srv.page_of  # a host hit is not copied back to a device page


def test_streaming_slots_pin_host_pages_not_device_pages():
    """P = S = 2: two slots stream from the host while both device pages are free to be refilled by new garments."""
    srv = _host_server(S=2, T=3, P=2, Q=4)
    for g in "ABCD":
        srv.submit(_req(g))
    srv.run()                                                # C, D on the device; A..D on the host
    assert set(srv.page_of) == {"C", "D"} and set(srv.host_page_of) == set("ABCD")
    srv.submit(_req("A", cloth=False))
    srv.submit(_req("B", cloth=False))
    srv.step()
    assert srv.den.page == [None, None] and srv.den.host_page == [0, 1]
    assert sum(srv.pins.values()) == 0 and srv.host_pins == {0: 1, 1: 1}
    srv.submit(_req("E"))                                    # waits for a slot; then a miss fills an unpinned page
    srv.run()
    assert "E" in srv.page_of and srv.stats["garment_host_hits"] == 2
    _check(srv)


def test_lru_in_each_tier():
    srv = _host_server(S=2, T=2, P=2, Q=2)
    for g in "WX":
        srv.submit(_req(g))
    srv.run()                                                # device [W, X], host [W, X]
    srv.submit(_req("W", cloth=False))                       # a device hit reorders the device LRU only
    srv.run()
    srv.submit(_req("Z"))                                    # device victim X, host victim W
    srv.run()
    assert set(srv.page_of) == {"W", "Z"} and set(srv.host_page_of) == {"X", "Z"}
    assert srv.stats["garment_page_evictions"] == 1 and srv.stats["garment_host_evictions"] == 1
    srv.submit(_req("X", cloth=False))                       # a host hit: X becomes the most recent host page
    srv.run()
    srv.submit(_req("Y"))                                    # host victim Z, not X; device victim W
    srv.run()
    assert set(srv.host_page_of) == {"X", "Y"} and set(srv.page_of) == {"Z", "Y"}
    _check(srv)


def test_write_through_is_skipped_when_every_host_page_is_pinned():
    srv = _host_server(S=2, T=3, P=2, Q=1)
    srv.submit(_req("A"))
    srv.run()
    srv.host_pins[srv.host_page_of["A"]] += 1               # as a slot streaming from A's host page pins it
    srv.submit(_req("B"))
    srv.step()
    assert srv.stats["garment_host_skipped"] == 1 and srv.stats["garment_host_writes"] == 1
    assert srv.host_page_of == {"A": 0} and srv.den.content[srv.page_of["B"]] == "B"   # the device page serves
    srv.run()
    srv.host_pins[0] -= 1
    srv.submit(_req("C"))                                    # unpinned again: C's write-through evicts A
    srv.run()
    assert srv.host_page_of == {"C": 0} and srv.stats["garment_host_evictions"] == 1


def test_stats_count_hits_writes_and_streamed_rows():
    srv = _host_server(S=2, T=3, P=2, Q=3)
    for g in "AB":
        srv.submit(_req(g))
    srv.run()
    srv.submit(_req("C"))                                    # A leaves the device
    srv.run()
    srv.submit(_req("A", cloth=False))                       # streams all 3 rows: 1 at admission, 2 after steps 0, 1
    srv.run()
    s = srv.stats
    assert (s["garment_page_fills"], s["garment_host_writes"], s["garment_host_hits"]) == (3, 3, 1)
    assert s["garment_rows_streamed"] == 3 and s["garment_bytes_streamed"] == 30
    assert s["garment_host_skipped"] == 0 and s["garment_host_evictions"] == 0 and s["images"] == 4


def test_host_tier_off_adds_no_stats_and_no_calls():
    from test_continuous_pool_cpu import _pool_fake_server
    srv = _pool_fake_server(S=2, T=2, P=2)
    for g in "ABCA":
        srv.submit(_req(g, cloth=g not in srv.garments))
    srv.run()
    assert not any(k.startswith("garment_host") or k.endswith("_streamed") for k in srv.stats)
    assert srv.host_page_of == {} and srv.free_host_pages == []


# ------------------------------------------------------------------------------------------------------------------
# budgets and refusals
# ------------------------------------------------------------------------------------------------------------------
def _engine(symbols=ROWS_SYMBOLS + ("b200vton_quantize_kv_e4m3", "b200vton_attention_kv8")):
    L = types.SimpleNamespace(has_symbol=lambda n: n in symbols, nchw_to_nhwc=lambda *a, **k: None)
    return types.SimpleNamespace(L=L, device=torch.device("cpu"), ch=(8, 16),
                                 blocks=lambda: [_Blk(16), _Blk(16), _Blk(8)],
                                 encode_context=lambda *a, **k: None)


def test_budgets_and_refusals(monkeypatch):
    from idm_vton_b200 import denoise as D
    from idm_vton_b200 import lib
    from idm_vton_b200.serving import ContinuousTryOnServer
    pipe, _, _ = _cpu_pipe(_schedulers()["ddpm"][0])
    with pytest.raises(ValueError, match="needs garment_kv_bytes"):
        ContinuousTryOnServer(pipe, height=32, width=32, slots=2, garment_kv_host_bytes=1 << 30)
    pipe.unet.engine = _engine
    page = 3 * (2 * (8 * 8 * 32 * 2) + 16 * 16 * 16 * 2)   # 3 steps at 16x16 latents (32x32 pixels)
    registered = []
    monkeypatch.setattr(D, "_host_register", lambda t: registered.append(t) or True)
    monkeypatch.setattr(D, "_host_unregister", lambda t: registered.pop(next(i for i, x in enumerate(registered) if x is t)))
    lib.load()
    n0 = lib.launch_count()
    srv = ContinuousTryOnServer(pipe, height=32, width=32, slots=2, num_inference_steps=3, garment_kv_bytes=2 * page,
                                garment_kv_host_bytes=page - 1)
    srv.submit(_req("A"))
    with pytest.raises(ValueError, match=f"holds no garment K/V page of {page} bytes"):
        srv.step()
    assert registered == [] and lib.launch_count() == n0
    srv = ContinuousTryOnServer(pipe, height=32, width=32, slots=2, num_inference_steps=3, garment_kv_bytes=2 * page,
                                garment_kv_host_bytes=3 * page + page // 2)
    assert srv._pages(3) == 2 and srv._host_pages(3) == 3
    # a refused page-lock: RuntimeError naming the bytes, nothing stays registered, no launch
    monkeypatch.setattr(D, "_host_register", lambda t: len(registered) < 2 and (registered.append(t) or True))
    srv.submit(_req("A"))
    with pytest.raises(RuntimeError, match=f"page-lock {3 * page} bytes"):
        srv.step()
    assert registered == [] and lib.launch_count() == n0


def _slot_den(monkeypatch, S=2, P=2, Q=2, T=4, fmt="fp16"):
    from idm_vton_b200 import denoise as D
    from idm_vton_b200.scheduler import DDPMScheduler
    registered = []
    monkeypatch.setattr(D, "_host_register", lambda t: registered.append(t) or True)
    monkeypatch.setattr(D, "_host_unregister", lambda t: registered.pop(next(i for i, x in enumerate(registered) if x is t)))
    eng = _engine()
    eng.garment_kv_format = fmt
    sch = DDPMScheduler()
    sch.set_timesteps(T)
    den = D.SlotDenoiser(eng, _engine(), S, pages=P, host_pages=Q)
    den.configure(sch, sch.timesteps, 4, 4)
    return den, registered


@pytest.mark.parametrize("fmt", ["fp16", "fp8"])
def test_pool_and_host_shapes_and_ring_rows(monkeypatch, fmt):
    from idm_vton_b200.denoise import SlotDenoiser, kv_parts
    den, registered = _slot_den(monkeypatch, S=3, P=3, Q=2, T=5, fmt=fmt)
    ring = 3 * 5
    assert den.ring == ring and [kv_parts(p)[0].shape[0] for p in den.pool] == [ring + 6] * 3
    assert [kv_parts(h)[0].shape[0] for h in den.host.blocks] == [10] * 3
    assert all(tuple(a.shape[1:]) == tuple(b.shape[1:]) and a.dtype == b.dtype and b.device.type == "cpu"
               for p, h in zip(den.pool, den.host.blocks) for a, b in zip(kv_parts(p), kv_parts(h)))
    assert len(registered) == 3 * len(kv_parts(den.pool[0]))
    assert den.host.bytes == sum(b.numel() * b.element_size() for h in den.host.blocks for b in kv_parts(h))
    # rows: a device page, a streaming slot at odd and even steps, an idle slot
    den.page, den.host_page = [2, None, None], [None, 1, None]
    assert den.kv_rows([3, 0, None]) == [2 * 5 + 3, ring + 2 + 0, -1]
    assert den.kv_rows([None, 3, None]) == [-1, ring + 2 + 1, -1]
    den.host_page = [None, None, 0]
    den.page = [None, None, None]
    assert den.kv_rows([None, None, 4]) == [-1, -1, ring + 4]
    den.page = [3, None, None]
    with pytest.raises(ValueError, match=rf"outside \[-1, {ring}\)"):     # a page past P never reads the ring
        den.kv_rows([0, None, None])
    den.release_host()
    assert registered == [] and den.host is None
    with pytest.raises(ValueError, match="needs pool mode"):
        SlotDenoiser(_engine(), _engine(), 2, host_pages=1)
    # the host tier off: the parent's pool shapes
    plain = SlotDenoiser(_engine(), _engine(), 3, pages=3)
    plain.configure(*_sched(5), 4, 4)
    assert [tuple(p.shape) for p in plain.pool] == [(15, 4, 32), (15, 4, 32), (15, 16, 16)] and plain.host is None


def _sched(T):
    from idm_vton_b200.scheduler import DDPMScheduler
    sch = DDPMScheduler()
    sch.set_timesteps(T)
    return sch, sch.timesteps


# ------------------------------------------------------------------------------------------------------------------
# stream and event order, with recorded streams and events
# ------------------------------------------------------------------------------------------------------------------
class _Recorder:
    def __init__(self):
        self.log, self.current = [], "main"
        self.n = 0

    def install(self, monkeypatch):
        rec = self

        class Ev:
            def __init__(self, *a, **k):
                rec.n += 1
                self.name = f"ev{rec.n}"

            def record(self, stream=None):
                rec.log.append(("record", self.name, rec.current if stream is None else stream.name))

        class Stream:
            def __init__(self, device=None):
                rec.n += 1
                self.name = f"s{rec.n}"

            def wait_event(self, ev):
                rec.log.append(("wait", self.name, ev.name))

            def wait_stream(self, other):
                rec.log.append(("wait_stream", self.name, other.name))

            def synchronize(self):
                rec.log.append(("sync", self.name))

        main = Stream()
        main.name = "main"

        @contextlib.contextmanager
        def stream(s):
            old, rec.current = rec.current, s.name
            try:
                yield
            finally:
                rec.current = old
        monkeypatch.setattr(torch.cuda, "Event", Ev)
        monkeypatch.setattr(torch.cuda, "Stream", Stream)
        monkeypatch.setattr(torch.cuda, "stream", stream)
        monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: main)


def test_ring_rows_and_event_order(monkeypatch):
    from idm_vton_b200 import denoise as D
    rec = _Recorder()
    rec.install(monkeypatch)
    den, _ = _slot_den(monkeypatch, S=2, P=2, Q=2, T=4)
    monkeypatch.setattr(D, "hoisted_garment_kv", lambda *a, **k: rec.log.append(("fill", rec.current)))
    den._run = lambda use_graph, name, *rows: (den._upload(*rows), rec.log.append(("replay", rec.current)))[1]
    den.ctx_t = []
    for h in den.host.blocks:                                # host page q, row i holds 100 q + i
        h.copy_((100 * torch.arange(2).repeat_interleave(4) + torch.arange(4).repeat(2)).view(8, 1, 1).expand_as(h))
    for p in den.pool:
        p.fill_(-1)
    ring = den.ring
    # a fill, its write-through, then a refill of that page: the refill waits for the write-through's event
    den.fill_page(0, torch.zeros(1, 4, 4, 4), torch.zeros(1, 77, 8))
    rec.log.clear()
    den.write_through(0, 1)
    wt = rec.log
    assert wt[0][0] == "record" and wt[0][2] == "main" and wt[1] == ("wait", "s2" if False else wt[1][1], wt[0][1])
    write_stream, done = wt[1][1], wt[-1][1]
    assert wt[-1] == ("record", done, write_stream) and ("wait_stream", write_stream, wt[2][2]) == wt[2]
    rec.log = []
    den.fill_page(0, torch.zeros(1, 4, 4, 4), torch.zeros(1, 77, 8))
    assert rec.log == [("wait", "main", done), ("fill", "main")]
    rec.log = []
    den.fill_page(0, torch.zeros(1, 4, 4, 4), torch.zeros(1, 77, 8))
    assert rec.log == [("fill", "main")]                     # once waited for, not again
    for h in den.host.blocks:                                # the write-through's rows, overwritten for the next check
        h.copy_((100 * torch.arange(2).repeat_interleave(4) + torch.arange(4).repeat(2)).view(8, 1, 1).expand_as(h))
    # slot 1 streams host page 1: the first row at admission, after the latest replay (none yet)
    den._host_written.clear()
    rec.log = []
    den.page[1], den.host_page[1] = None, 1
    den._stream_rows([(1, 0)], after_last_step=True)
    ring_stream = den._side["ring"].name
    assert all(p[ring + 2].eq(100).all() for p in den.pool) and all(p[ring + 3].eq(-1).all() for p in den.pool)
    assert rec.log == [("record", den._side["ring_ready"].name, ring_stream)]
    assert den.take_streamed() == (1, sum(p[0].numel() * 2 for p in den.pool)) and den.take_streamed() == (0, 0)
    # step 0: the replay waits for the ring; then step 1's row goes to ring row 1, after no earlier replay
    rec.log = []
    den.step([None, 0])
    replayed = den._side["replayed"]
    assert rec.log[0] == ("wait", "main", den._side["ring_ready"].name) and rec.log[1] == ("replay", "main")
    assert rec.log[2] == ("record", replayed[0].name, "main")
    assert rec.log[3:] == [("record", den._side["ring_ready"].name, ring_stream)]   # replay 0 is the first
    assert all(p[ring + 3].eq(101).all() for p in den.pool)
    # step 1 (replay 1): step 2's row goes to ring row 0 after replay 0, the step that last read it
    rec.log = []
    den.step([None, 1])
    assert rec.log[:3] == [("wait", "main", den._side["ring_ready"].name), ("replay", "main"),
                           ("record", replayed[1].name, "main")]
    assert rec.log[3] == ("wait", ring_stream, replayed[0].name)
    assert all(p[ring + 2].eq(102).all() for p in den.pool)
    rec.log = []
    den.step([None, 2])                                      # replay 2: row 3 into ring row 1, after replay 1
    assert rec.log[3] == ("wait", ring_stream, replayed[1].name) and all(p[ring + 3].eq(103).all() for p in den.pool)
    assert den.rows.tolist() == [-1, ring + 2]               # the row table of step 2
    rec.log = []
    den.step([None, 3])                                      # the last step: nothing more to stream
    assert [e[0] for e in rec.log] == ["wait", "replay", "record"] and den.take_streamed()[0] == 3
    assert den.rows.tolist() == [-1, ring + 3]
    # a slot admitted now waits for the latest replay (3) before its first row
    rec.log = []
    den.host_page[0] = 0
    den._stream_rows([(0, 0)], after_last_step=True)
    assert rec.log[0] == ("wait", ring_stream, replayed[1].name) and all(p[ring].eq(0).all() for p in den.pool)
