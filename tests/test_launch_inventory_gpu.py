"""Launch-inventory parity: every distinct kernel call of full-size try-on steps, replayed in isolation against float64.

The SDXL-width engines (random fp16 weights, the `full` pattern of tests/test_fullsize_gpu.py) run, in eager mode, with
every op wrapper of idm_vton_b200.lib recorded (tests/helpers/launch_inventory.py):
  (a) one CFG step at 128x96 latents, B = 2 (garment forward + try-on forward, as _engine_step);
  (b) the same at 128x128, B = 1;
  (c) TryOnDenoiser(hoist_garment=True), a 30-step DDPM plan: its hoisting pass and its first step;
  (d) one hoisted step at 33x25 person latents with a 32x24 garment (the resolution suite's SDXL-width case):
      upsample_nearest and ragged convolution boxes;
  (e) SlotDenoiser in pool mode, three slots: two at different steps of their own garment page, one idle (row -1);
  (f) the opt-in modes at 128x96, B = 2: UNetEngine(fp8=True) for one step, and FP8 garment K/V for one hoisted step.
Each distinct signature is then replayed on fresh operands with its recorded shapes, strides, offsets, aliasing,
scalars and tables, and compared with the float64 restatement of the same op:
  * GEMM / convolution on grid operands: bit-identical (the fp32 sums are exact), TOL_EPI_ACT with GEGLU / GELU; large M
    on a row sample covering every 128-row tile; the GEGLU weight packed at the width the engine packed it for;
  * e4m3 GEMM: the float64 product of the same e4m3 operands, test_fp8_gpu's bound per rounding point;
  * attention / cross-attention / attention_rows / kv8: per (sample, head), TOL_ATTN / TOL_ATTN_IP, with mutants
    (segment 1 of the neighbouring row, the uncond half without its zero tokens, the IP rounding); kv8 launches also
    bit-identical to the fp16 kernel on the dequantized K/V;
  * GroupNorm / LayerNorm: float64 within TOL_NORM16, with mutants (eps dropped, the straddling group read in source 0's
    layout); layernorm_e4m3 and quantize_kv_e4m3 bit for bit by their rules;
  * layout / resampling kernels bit-identical to torch; timestep embedding and skinny linears within one fp16 ulp;
  * the CFG step kernels within the solver / schedule TOL, with a mutant each.
One line per signature is printed (`pytest -s`): family, key shape, tile width, error, gate and the smallest mutant
ratio. The coverage assertion names every family the inventory must hold."""
import collections
import importlib.util
import os
import time

import pytest
import torch
import torch.nn.functional as F

from test_kernel_edges_gpu import (TOL_ATTN, TOL_ATTN_IP, TOL_EPI_ACT, TOL_NORM16, U16, attn_head_ref, conv3x3_acc,
                                   gelu64, gemm_epilogue_ref, group_norm64, ip_ref, quick_gelu64, r16, rel_err)
from test_schedule_cpu import cfg_rescale_ddpm_ref
from test_solvers_cpu import TOL, cfg_solver_ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _helper(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tests", "helpers", f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


LI = _helper("launch_inventory")
Q = _helper("fp8_ref")
K8 = _helper("kv8_ref")
GEMM_TOL_E4M3 = 2.0 ** -10      # tests/test_fp8_gpu.py GEMM_TOL: one fp16 ulp of the output per epilogue rounding point
DEV = "cuda"


# ------------------------------------------------------------------------------------------------------------------
# recording
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def inventory():
    """Builds the engines (recording the GEGLU packing width of every FF1 weight), records runs (a)-(f) and returns
    {run: {signature: calls}} plus the run notes."""
    from test_fullsize_gpu import _engine_step, _forward_inputs
    from idm_vton_b200 import engine as E
    from idm_vton_b200 import lib as L
    from idm_vton_b200 import unet as U
    from idm_vton_b200.denoise import SlotDenoiser, TryOnDenoiser
    from idm_vton_b200.scheduler import DDPMScheduler
    from oracle import loop_ref as LR
    t0 = time.time()
    pack_bn = {}
    with pytest.MonkeyPatch.context() as mp:
        orig_pack, orig_q = E.pack_geglu, L.quantize_rows_e4m3

        def pack(w, b, bn):
            wp, bp = orig_pack(w, b, bn)
            pack_bn[wp.data_ptr()] = bn
            return wp, bp

        def quant(w):
            q, s = orig_q(w)
            if w.data_ptr() in pack_bn:
                pack_bn[q.data_ptr()] = pack_bn[w.data_ptr()]
            return q, s

        mp.setattr(E, "pack_geglu", pack)
        mp.setattr(L, "quantize_rows_e4m3", quant)
        sd_t = U.random_state_dict(E.SDXL_TRYON, seed=11, device=DEV)
        sd_g = U.random_state_dict(E.SDXL_GARMENT, seed=22, device=DEV)
        env = dict(eng_t=E.UNetEngine(E.SDXL_TRYON, sd_t, "tryon"), eng_g=E.UNetEngine(E.SDXL_GARMENT, sd_g, "garment"))
    runs, notes = {}, {}
    sch = DDPMScheduler()
    sch.set_timesteps(30)

    def record(name, fn):
        with pytest.MonkeyPatch.context() as mp:
            rec = LI.Recorder(L, mp, pack_bn)
            assert not rec.missing, f"library binding without {rec.missing}"
            with torch.no_grad():
                fn()
            torch.cuda.synchronize()
        runs[name] = rec.sigs
        torch.cuda.empty_cache()

    def hoisted(den, inp, noise):
        den.prepare(**inp, guidance_scale=2.0)
        den.set_step_tables(sch, sch.timesteps)
        den.step(0, noise, use_graph=False)
        return den.window

    inp2 = _forward_inputs(E.SDXL_TRYON, E.SDXL_GARMENT, 2, 128, 96, seed=9)
    noise2 = torch.randn(2, 4, 128, 96, generator=torch.Generator().manual_seed(5)).half().cuda()
    record("a", lambda: _engine_step(env, inp2, 967, 2, 128, 96))
    record("b", lambda: _engine_step(env, _forward_inputs(E.SDXL_TRYON, E.SDXL_GARMENT, 1, 128, 128, seed=8), 301, 1,
                                     128, 128))
    notes["a"] = notes["b"] = dict(Bg=None)

    def run_c():
        notes["c"] = dict(Bg=2, window=hoisted(TryOnDenoiser(env["eng_t"], env["eng_g"]), inp2, noise2))
    record("c", run_c)

    def run_d():
        B, h, w, hg, wg = 2, 33, 25, 32, 24          # tests/test_resolution_gpu.py, test_sdxl_width_odd_sizes_vs_oracle
        inp = LR.synth_loop_inputs(E.SDXL_TRYON, E.SDXL_GARMENT, B, h, w, seed=17)
        inp["cloth_latents"] = torch.randn(B, 4, hg, wg, generator=torch.Generator().manual_seed(18)) * 0.5
        inp = {k: (v.half().float() if k != "add_time_ids" else v).cuda() for k, v in inp.items()}
        noise = torch.randn(B, 4, h, w, generator=torch.Generator().manual_seed(6)).half().cuda()
        notes["d"] = dict(Bg=B, window=hoisted(TryOnDenoiser(env["eng_t"], env["eng_g"]), inp, noise))
    record("d", run_d)

    def run_e():
        den = SlotDenoiser(env["eng_t"], env["eng_g"], 3, pages=3)
        den.configure(sch, sch.timesteps, 128, 96, guidance_scale=2.0)
        for s, seed in ((0, 3), (1, 4)):
            inp = _forward_inputs(E.SDXL_TRYON, E.SDXL_GARMENT, 1, 128, 96, seed=seed)
            den.fill_page(s, inp["cloth_latents"], inp["text_embeds_cloth"])
            den.admit(s, latents=inp["latents"], mask=inp["mask"], masked_image_latents=inp["masked_image_latents"],
                      pose_latents=inp["pose_latents"], cloth_latents=inp["cloth_latents"],
                      prompt_embeds=inp["prompt_embeds"], add_text_embeds=inp["add_text_embeds"],
                      add_time_ids=inp["add_time_ids"], image_embeds=inp["image_embeds"],
                      text_embeds_cloth=inp["text_embeds_cloth"], page=s)
        den.step([3, 10, None], {0: noise2[:1], 1: noise2[1:]}, use_graph=False)
        notes["e"] = dict(Bg=None, slots="steps 3 / 10 / idle")
    record("e", run_e)

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(E, "pack_geglu", pack)
        mp.setattr(L, "quantize_rows_e4m3", quant)
        env8 = dict(eng_t=E.UNetEngine(E.SDXL_TRYON, sd_t, "tryon", fp8=True), eng_g=env["eng_g"])
    record("f_fp8_linears", lambda: _engine_step(env8, inp2, 501, 2, 128, 96))
    del env8
    torch.cuda.empty_cache()

    def run_f2():
        env["eng_t"].garment_kv_format = "fp8"
        try:
            notes["f_fp8_kv"] = dict(Bg=2, window=hoisted(TryOnDenoiser(env["eng_t"], env["eng_g"]), inp2, noise2))
        finally:
            env["eng_t"].garment_kv_format = "fp16"
    record("f_fp8_kv", run_f2)
    del env
    torch.cuda.empty_cache()
    print(f"[inventory] recorded in {time.time() - t0:.1f} s")
    for r, sigs in runs.items():
        print(f"[inventory] run {r}: {len(sigs)} unique signatures, {sum(sigs.values())} calls; {notes.get(r)}")
    yield dict(runs=runs, notes=notes)


# ------------------------------------------------------------------------------------------------------------------
# replay: one function per family, each returning (key shape, tile width, err, gate, {mutant: err}, exact)
# ------------------------------------------------------------------------------------------------------------------
def _rows_t(M):
    return torch.tensor(LI.sample_rows(M), dtype=torch.long, device=DEV)


def _fill(t, x):
    t.copy_(x.to(t.dtype).view(t.shape))


def _replay_gemm(sig, o, seed):
    from idm_vton_b200 import lib as L
    from idm_vton_b200.engine import pack_geglu
    a, w = o["a"], o["w"]
    M, K = a.shape
    N = w.shape[0]
    geglu = bool(o["geglu"])
    _fill(a, LI.grid_dev(a.shape, 1.0, seed, DEV))
    w_u = LI.grid_dev(w.shape, 0.25, seed + 1, DEV)
    b_u = LI.randn_dev((N,), seed + 2, DEV) if o["bias"] is not None else None
    if geglu:
        wp, bp = pack_geglu(w_u, b_u, o.get("pack_bn") or o["force_bn"] % 1000)
        _fill(w, wp)
        if b_u is not None:
            _fill(o["bias"], bp)
    else:
        _fill(w, w_u)
        if b_u is not None:
            _fill(o["bias"], b_u)
    if o["residual"] is not None:
        _fill(o["residual"], LI.randn_dev(o["residual"].shape, seed + 3, DEV))
    if o["rowvec"] is not None:
        _fill(o["rowvec"], LI.randn_dev(o["rowvec"].shape, seed + 4, DEV))
    rows = _rows_t(M)
    ins = {k: (o[k][rows].clone() if k in ("a", "residual") else o[k].clone()) if o[k] is not None else None
           for k in ("a", "bias", "residual", "rowvec")}
    out = L.gemm(o["a"], o["w"], bias=o["bias"], residual=o["residual"], rowvec=o["rowvec"],
                 rows_per_sample=o["rows_per_sample"], geglu=geglu, gelu=o["gelu"], out=o["out"], force_bn=o["force_bn"],
                 quick_gelu=o["quick_gelu"])
    acc = ins["a"].double() @ w_u.double().t()
    rv, rps = None, 0
    if ins["rowvec"] is not None:
        rps = o["rows_per_sample"]
        rv = ins["rowvec"][rows // rps if rps else torch.zeros_like(rows)]
        rps = 1
    act = gelu64 if o["gelu"] else quick_gelu64 if o["quick_gelu"] else None
    if geglu:
        v = gemm_epilogue_ref(acc, b_u)
        ref = r16(v[:, :N // 2] * r16(gelu64(v[:, N // 2:])))
    else:
        ref = gemm_epilogue_ref(acc, ins["bias"], act, rv, rps, ins["residual"])
    got = out[rows]
    gate = TOL_EPI_ACT if (geglu or act is not None) else 0.0
    key = f"M={M} N={N} K={K}" + (" bias" if o["bias"] is not None else "") + (" res" if o["residual"] is not None else "") \
        + (" geglu" if geglu else "") + (" gelu" if act is not None else "")
    return key, LI.pick_bn(N, M, geglu, o["force_bn"]), rel_err(got, ref), gate, {}, torch.equal(got.double(), ref)


def _replay_gemm_e4m3(sig, o, seed):
    from idm_vton_b200 import lib as L
    from idm_vton_b200.engine import pack_geglu
    M, K = o["a_q"].shape
    N = o["w_q"].shape[0]
    geglu = bool(o["geglu"])
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = (torch.randn(M, K, generator=g, device=DEV) * 2.0 ** torch.randint(-6, 3, (M, 1), generator=g, device=DEV)).half()
    w = (torch.randn(N, K, generator=g, device=DEV) / K ** 0.5).half()
    bias = (0.5 * torch.randn(N, generator=g, device=DEV)).half() if o["bias"] is not None else None
    if geglu:
        w, bias = pack_geglu(w, bias, o.get("pack_bn") or o["force_bn"] % 1000)
    qa, sa = Q.quantize_rows(a)
    qw, sw = Q.quantize_rows(w)
    _fill(o["a_q"], qa); _fill(o["a_scale"], sa); _fill(o["w_q"], qw); _fill(o["w_scale"], sw)
    if bias is not None:
        _fill(o["bias"], bias)
    res = None
    if o["residual"] is not None:
        _fill(o["residual"], LI.randn_dev(o["residual"].shape, seed + 3, DEV))
    rows = _rows_t(M)
    if o["residual"] is not None:
        res = o["residual"][rows].clone()
    out = L.gemm_e4m3(o["a_q"], o["a_scale"], o["w_q"], o["w_scale"], bias=o["bias"], residual=o["residual"],
                      geglu=geglu, out=o["out"], force_bn=o["force_bn"])
    ref = Q.epilogue(Q.scaled_acc(qa[rows], sa[rows], qw, sw), bias, res, geglu_bn=o["force_bn"] % 1000 if geglu else 0)
    gate = (2 if (res is not None or geglu) else 1) * GEMM_TOL_E4M3
    key = f"M={M} N={N} K={K}" + (" res" if res is not None else "") + (" geglu" if geglu else "")
    return key, LI.pick_bn(N, M, geglu, o["force_bn"]), rel_err(out[rows], ref), gate, {}, False


def _conv_patches(x, rows, Ho, Wo, stride):
    """The 3x3 input neighbourhood of each sampled output pixel (zero outside the image): conv3x3_acc of the patch at
    its centre is the output pixel's accumulator."""
    B, H, W, C = x.shape
    b, rem = rows // (Ho * Wo), rows % (Ho * Wo)
    y, xx = rem // Wo, rem % Wo
    d = torch.arange(3, device=x.device) - 1
    iy = y[:, None] * stride + d[None, :]
    ix = xx[:, None] * stride + d[None, :]
    ok = ((iy >= 0) & (iy < H))[:, :, None] & ((ix >= 0) & (ix < W))[:, None, :]
    p = x[b[:, None, None], iy.clamp(0, H - 1)[:, :, None], ix.clamp(0, W - 1)[:, None, :]]
    return p * ok[..., None].to(p.dtype), b


def _replay_conv(sig, o, seed):
    from idm_vton_b200 import lib as L
    from idm_vton_b200.engine import pack_conv3x3
    x = o["x"]
    B, H, W, Cin = x.shape
    Cout = o["w_packed"].shape[1]
    st = o["stride"]
    _fill(x, LI.grid_dev(x.shape, 1.0, seed, DEV))
    w = LI.grid_dev((Cout, Cin, 3, 3), 0.25, seed + 1, DEV)
    _fill(o["w_packed"], pack_conv3x3(w))
    for i, k in enumerate(("bias", "temb", "bias_sc", "residual")):
        if o[k] is not None:
            _fill(o[k], LI.randn_dev(o[k].shape, seed + 2 + i, DEV))
    for i, k in enumerate(("sc0", "sc1")):
        if o[k] is not None:
            _fill(o[k], LI.grid_dev(o[k].shape, 1.0, seed + 6 + i, DEV))
    if o["w_sc"] is not None:
        _fill(o["w_sc"], LI.grid_dev(o["w_sc"].shape, 0.25, seed + 8, DEV))
    Ho, Wo = (H - 1) // st + 1, (W - 1) // st + 1
    rows = _rows_t(B * Ho * Wo)
    patches, bidx = _conv_patches(x, rows, Ho, Wo, st)
    snap = {k: (o[k].clone() if o[k] is not None else None) for k in ("bias", "temb", "bias_sc", "w_sc")}
    res = o["residual"].reshape(-1, Cout)[rows].clone() if o["residual"] is not None else None
    sc = None
    if o["sc0"] is not None:
        cat = torch.cat([o["sc0"], o["sc1"]], -1) if o["sc1"] is not None else o["sc0"]
        sc = cat.reshape(-1, cat.shape[-1])[rows].clone()
    out = L.conv3x3(x, o["w_packed"], bias=o["bias"], temb=o["temb"], sc0=o["sc0"], sc1=o["sc1"], w_sc=o["w_sc"],
                    bias_sc=o["bias_sc"], residual=o["residual"], out=o["out"], force_bn=o["force_bn"], stride=st)
    acc = conv3x3_acc(patches, w)[:, 1, 1, :]
    assert res is None or snap["temb"] is None, "conv with both temb and residual: no restatement"
    if sc is not None:
        res = r16(sc.double() @ snap["w_sc"].double().t() + snap["bias_sc"].double())
    rv = snap["temb"][bidx] if snap["temb"] is not None else None
    ref = gemm_epilogue_ref(acc, snap["bias"], None, rv, 1 if rv is not None else 0, res)
    got = out.reshape(-1, Cout)[rows]
    key = f"B={B} {H}x{W} Cin={Cin} Cout={Cout}" + (" s2" if st == 2 else "") + (" temb" if rv is not None else "") \
        + (f" shortcut {o['sc0'].shape[-1]}+{o['sc1'].shape[-1] if o['sc1'] is not None else 0}" if sc is not None else "") \
        + (" res" if o["residual"] is not None else "")
    return key, o["force_bn"] or "auto", rel_err(got, ref), 0.0, {}, torch.equal(got.double(), ref)


def _attn_core(o, seed, kind):
    """Fills q / k0 / v0 / segment 1, runs the kernel, and compares per (sample, head) on sampled query rows with the
    truth and the mutants. kind: attention | attention_rows | attention_kv8."""
    from idm_vton_b200 import lib as L
    q, k0, v0 = o["q"], o["k0"], o["v0"]
    B, Nq = q.shape[0], q.shape[1]
    H = o["heads"]
    C = 64 * H
    for i, k in enumerate(("q", "k0", "v0")):
        _fill(o[k], LI.randn_dev(o[k].shape, seed + i, DEV))
    deq = None
    if kind == "attention_kv8":
        kq, e = o["kv1"]
        B1, N1 = kq.shape[0], kq.shape[1]
        kv = LI.randn_dev(kq.shape, seed + 3, DEV)
        qq, ee = K8.quantize(kv, H)
        kq.copy_(qq)
        e.zero_()
        e[:, :, :N1].copy_(ee.to(torch.int8))
        deq = K8.dequantize(kq, e)
        k1, v1 = deq[..., :C], deq[..., C:]
    else:
        k1, v1 = o["k1"], o["v1"]
        if k1 is not None:
            _fill(k1, LI.randn_dev(k1.shape, seed + 3, DEV))
            _fill(v1, LI.randn_dev(v1.shape, seed + 4, DEV))
        B1 = k1.shape[0] if k1 is not None else 0
        N1 = k1.shape[1] if k1 is not None else o.get("n1", 0)
    acc = bool(o["accumulate"])
    if acc:
        _fill(o["out"], LI.randn_dev(o["out"].shape, seed + 5, DEV))
    before = o["out"].clone() if acc else None
    rows_tab = o.get("kv1_rows")
    rows_list = rows_tab.tolist() if rows_tab is not None else None
    base = int(o["kv1_base"].item()) if o.get("kv1_base") is not None else 0
    mod = o.get("kv1_mod", 0) or 0
    scale = o["scale"] if o["scale"] is not None else 64 ** -0.5
    if kind == "attention":
        out = L.attention(q, k0, v0, k1, v1, n1=o["n1"], kv1_off=o["kv1_off"], heads=H, scale=o["scale"],
                          accumulate=acc, out=o["out"], kv1_mod=mod, kv1_base=o["kv1_base"])
    elif kind == "attention_rows":
        out = L.attention_rows(q, k0, v0, k1, v1, o["kv1_rows"], kv1_off=o["kv1_off"], heads=H, scale=o["scale"],
                               accumulate=acc, out=o["out"])
    else:
        out = L.attention_kv8(q, k0, v0, L.GarmentKV8(*o["kv1"]), kv1_off=o["kv1_off"], heads=H, scale=o["scale"],
                              accumulate=acc, out=o["out"], kv1_mod=mod, kv1_base=o["kv1_base"], kv1_rows=o["kv1_rows"])
    exact = None
    if kind == "attention_kv8":
        out = out.clone()
        if rows_tab is not None:
            o16 = L.attention_rows(q, k0, v0, k1, v1, rows_tab, kv1_off=o["kv1_off"], heads=H, scale=o["scale"])
        else:
            o16 = L.attention(q, k0, v0, k1, v1, kv1_off=o["kv1_off"], heads=H, scale=o["scale"], kv1_mod=mod,
                              kv1_base=o["kv1_base"])
        exact = torch.equal(out, o16)
    if B1:
        truth = LI.seg1_rows(B, o["kv1_off"], B1, mod, base, rows_list)
        nb = LI.neighbour_rows(B, o["kv1_off"], B1, truth, mod, base, rows_list)
    else:
        truth, nb = [None] * B, [None] * B
    qr = _rows_t(Nq)
    errs, merrs = [], collections.defaultdict(lambda: float("inf"))
    for b in range(B):
        for h in range(H):
            c = slice(64 * h, 64 * h + 64)

            def ref(row, n_zero):
                kk, vv = k0[b, :, c], v0[b, :, c]
                if row is not None:
                    kk, vv = torch.cat([kk, k1[row, :, c]]), torch.cat([vv, v1[row, :, c]])
                r = attn_head_ref(q[b, qr, c], kk, vv, scale, n_zero=n_zero)
                return r16(before[b, qr, c].double() + r16(r)) if acc else r
            nz = N1 if truth[b] is None else 0
            t = ref(truth[b], nz)
            errs.append(rel_err(out[b, qr, c], t))
            if nb[b] is not None:
                merrs["seg1 neighbour row"] = min(merrs["seg1 neighbour row"], rel_err(ref(nb[b], 0), t))
            if truth[b] is None and nz:
                merrs["uncond without zero tokens"] = min(merrs["uncond without zero tokens"], rel_err(ref(None, 0), t))
                merrs["n1-1 (shown only)"] = min(merrs["n1-1 (shown only)"], rel_err(ref(None, nz - 1), t))
    key = f"B={B} H={H} Nq={Nq} N0={k0.shape[1]} N1={N1} B1={B1} off={o['kv1_off']}" + \
        (f" mod={mod}" if mod else "") + (f" base={base}" if o.get("kv1_base") is not None else "") + \
        (f" rows={rows_list}" if rows_list is not None else "") + (" acc" if acc else "")
    return key, "-", max(errs), TOL_ATTN_IP if acc else TOL_ATTN, dict(merrs), exact


def _replay_cross(sig, o, seed):
    from idm_vton_b200 import lib as L
    q, kt, vt, ki, vi = (o[k] for k in ("q", "kt", "vt", "ki", "vi"))
    B, Nq = q.shape[0], q.shape[1]
    H = o["heads"]
    scale = o["scale"] if o["scale"] is not None else 64 ** -0.5
    s = o["ip_scale"]
    for i, k in enumerate(("q", "kt", "vt", "ki", "vi")):
        if o[k] is not None:
            _fill(o[k], LI.randn_dev(o[k].shape, seed + i, DEV))
    out = L.cross_attention(q, kt, vt, ki, vi, heads=H, scale=o["scale"], ip_scale=s, out=o["out"]).clone()
    qr = _rows_t(Nq)
    errs = []
    for b in range(B):
        for h in range(H):
            c = slice(64 * h, 64 * h + 64)
            ot = attn_head_ref(q[b, qr, c], kt[b, :, c], vt[b, :, c], scale)
            ref = ip_ref(ot, attn_head_ref(q[b, qr, c], ki[b, :, c], vi[b, :, c], scale), s) if ki is not None else ot
            errs.append(rel_err(out[b, qr, c], ref))
    merrs, exact = {}, None
    if ki is not None and s == 1.0:
        # exact softmax (q = 0: every score 0, P = 1, l = N) on grid values whose sums are exact in fp32, and an IP term
        # that nearly cancels the text term: only the rounding points decide, and O_t must be rounded before the sum
        q.zero_()
        vt_c, vi_c = LI.ip_cancel_values(vt.shape, vi.shape, seed + 7, DEV)
        _fill(vt, vt_c)
        _fill(vi, vi_c)
        out = L.cross_attention(q, kt, vt, ki, vi, heads=H, scale=o["scale"], ip_scale=s, out=o["out"])
        ot, oi = vt.double().mean(1, keepdim=True), vi.double().mean(1, keepdim=True)
        ref = ip_ref(ot, oi, s).expand(B, Nq, -1)
        e = rel_err(out, ref)
        errs.append(e)
        exact = e == 0.0
        merrs["O_t unrounded"] = rel_err(ip_ref(ot, oi, s, mutant="ot_unrounded"), ref[:, :1])
    key = f"B={B} H={H} Nq={Nq} Nt={kt.shape[1]} Ni={ki.shape[1] if ki is not None else 0} ip_scale={s}"
    return key, "-", max(errs), TOL_ATTN_IP if ki is not None else TOL_ATTN, merrs, exact


def _replay_groupnorm(sig, o, seed):
    from idm_vton_b200 import lib as L
    x0, x1 = o["x0"], o["x1"]
    B, C0 = x0.shape[0], x0.shape[-1]
    C1 = x1.shape[-1] if x1 is not None else 0
    _fill(x0, LI.gn_offset_dev(x0.shape, seed, DEV))
    if x1 is not None:
        _fill(x1, LI.gn_offset_dev(x1.shape, seed + 1, DEV))
    _fill(o["gamma"], LI.randn_dev(o["gamma"].shape, seed + 2, DEV))
    _fill(o["beta"], LI.randn_dev(o["beta"].shape, seed + 3, DEV))
    out = L.groupnorm(x0, o["gamma"], o["beta"], o["eps"], o["silu"], x1=x1, out=o["out"], ws=o["ws"])
    x0f = x0.reshape(B, -1, C0)
    act = F.silu if o["silu"] else (lambda v: v)

    def ref(xa, xb, eps):
        x = torch.cat([xa, xb.reshape(B, -1, C1)], -1) if xb is not None else xa
        return act(group_norm64(x, 32, o["gamma"], o["beta"], eps))
    truth = ref(x0f, x1, o["eps"])
    merrs = {"eps dropped": rel_err(ref(x0f, x1, 0.0), truth)}
    gs, straddle = LI.gn_groups(C0, C1)
    if x1 is not None and C1 != C0:                  # equal widths: source 0's layout is source 1's
        merrs["x1 in source 0's layout"] = rel_err(ref(x0f, LI.gn_x1_in_x0_layout(x1, C0), o["eps"]), truth)
    key = f"B={B} HW={x0f.shape[1]} C={C0}" + (f"+{C1} group {gs} ch" + (f", group {straddle} straddles" if straddle
                                                                         is not None else ", no straddle") if C1 else "")
    return key, "-", rel_err(out.reshape(B, -1, C0 + C1), truth), TOL_NORM16, merrs, None


def _replay_layernorm(sig, o, seed, e4m3=False):
    from idm_vton_b200 import lib as L
    x = o["x"]
    C = x.shape[-1]
    _fill(x, LI.randn_dev(x.shape, seed, DEV, scale=3.0, shift=1.0))
    _fill(o["gamma"], LI.randn_dev(o["gamma"].shape, seed + 1, DEV, scale=0.1, shift=1.0))
    if o["beta"] is not None:
        _fill(o["beta"], LI.randn_dev(o["beta"].shape, seed + 2, DEV, scale=0.1))
    x2 = x.reshape(-1, C)
    rows = _rows_t(x2.shape[0])
    ref = F.layer_norm(x2[rows].double(), (C,), o["gamma"].double(),
                       o["beta"].double() if o["beta"] is not None else None, o["eps"])
    exact = None
    if e4m3:
        q, s, y16 = L.layernorm_e4m3(x, o["gamma"], o["beta"], o["eps"], fp16_out=o["fp16_out"])
        y = L.layernorm(x, o["gamma"], o["beta"], o["eps"]).reshape(-1, C)
        qr, sr = Q.quantize_rows(y)
        exact = torch.equal(q.float(), qr) and torch.equal(s, sr) and (y16 is None or torch.equal(y16, y))
        got = y[rows]
    else:
        got = L.layernorm(x, o["gamma"], o["beta"], o["eps"], out=o["out"]).reshape(-1, C)[rows]
    return f"rows={x2.shape[0]} C={C}", "-", rel_err(got, ref), TOL_NORM16, {}, exact


def _replay_quantize_kv(sig, o, seed):
    from idm_vton_b200 import lib as L
    x = o["x"]
    q, e = o["out"]
    H = x.shape[-1] // 128
    _fill(x, LI.randn_dev(x.shape, seed, DEV, scale=4.0))
    L.quantize_kv_e4m3(x, L.GarmentKV8(q, e))
    qr, er = K8.quantize(x, H)
    ng = x.shape[1]
    exact = torch.equal(q.view(torch.uint8), qr.view(torch.uint8)) and torch.equal(e[:, :, :ng].int(), er)
    return f"rows={x.shape[0]} Ng={ng} 2C={x.shape[-1]}", "-", 0.0 if exact else float("inf"), 0.0, {}, exact


def _replay_skinny(sig, o, seed):
    from idm_vton_b200 import lib as L
    x, w = o["x"], o["w"]
    K = x.shape[1]
    _fill(x, LI.randn_dev(x.shape, seed, DEV))
    _fill(w, LI.randn_dev(w.shape, seed + 1, DEV, scale=K ** -0.5))
    for i, k in enumerate(("bias", "addend")):
        if o[k] is not None:
            _fill(o[k], LI.randn_dev(o[k].shape, seed + 2 + i, DEV))
    snap = {k: (o[k].clone() if o[k] is not None else None) for k in ("x", "w", "bias", "addend")}
    out = L.skinny_linear(x, w, o["bias"], in_silu=o["in_silu"], out_silu=o["out_silu"], addend=o["addend"], out=o["out"])
    xs = r16(F.silu(snap["x"].double())) if o["in_silu"] else snap["x"].double()
    y = xs @ snap["w"].double().t()
    y = r16(y + snap["bias"].double()) if snap["bias"] is not None else r16(y)
    if o["out_silu"]:
        y = r16(F.silu(y))
    if snap["addend"] is not None:
        y = r16(y + snap["addend"].double())
    err = rel_err(out, y)
    return f"M={x.shape[0]} K={K} N={w.shape[0]}", "-", err, 2 * U16, {}, None


def _replay_timestep(sig, o, seed):
    from idm_vton_b200 import lib as L
    v = o["values"]
    out = L.timestep_embedding(v, o["dim"], rows_repeat=o["rows_repeat"], out=o["out"])
    arg = LI.timestep_args(v, o["dim"]).double()
    ref = r16(torch.cat([torch.cos(arg), torch.sin(arg)], -1)).repeat(o["rows_repeat"], 1)
    # one fp16 ulp of the output's scale (|out| <= 1): the fp32 argument reaches ~1000, where one fp32 ulp of freq
    # (expf / logf of the kernel vs torch's) moves cos / sin by ~6e-5, several ulps of an output near zero
    ulps = ((out.double() - ref).abs().max() / LI.ulp16(ref.abs().max())).item()
    vals = sorted(set(v.tolist()))
    return f"n={v.numel()} dim={o['dim']} x{o['rows_repeat']} t={vals[:6]}", "-", ulps, 1.0, {}, None


def _replay_layout(sig, o, seed):
    from idm_vton_b200 import lib as L
    name = sig[0]
    if name in ("upsample2x", "upsample_nearest"):
        x = o["x"]
        _fill(x, LI.randn_dev(x.shape, seed, DEV))
        if name == "upsample2x":
            out = L.upsample2x(x, out=o["out"])
            ref = x.repeat_interleave(2, 1).repeat_interleave(2, 2)
        else:
            out = L.upsample_nearest(x, o["size"], out=o["out"])
            ref = F.interpolate(x.permute(0, 3, 1, 2).float(), size=tuple(o["size"]), mode="nearest").half() \
                .permute(0, 2, 3, 1)
        key = f"{tuple(x.shape)} -> {tuple(out.shape[1:3])}"
    elif name == "nhwc_to_nchw":
        src = o["src"]
        _fill(src, LI.randn_dev(src.shape, seed, DEV))
        out = L.nhwc_to_nchw(src, o["C"], out=o["out"])
        ref = src[..., :o["C"]].permute(0, 3, 1, 2)
        key = f"{tuple(src.shape)} C={o['C']}"
    else:
        src, dst = o["src"], o["dst"]
        _fill(src, LI.randn_dev(src.shape, seed, DEV, scale=3.0))
        _fill(dst, LI.randn_dev(dst.shape, seed + 1, DEV))
        ref = dst.clone()
        Bs, c0, Cs = src.shape[0], o["c_off"], src.shape[1]
        idx = torch.arange(dst.shape[0], device=DEV) % Bs
        val = src[idx].permute(0, 2, 3, 1)
        if name == "nchw_to_nhwc":
            L.nchw_to_nhwc(src, dst, c_off=c0)
        elif name == "nchw_to_nhwc_scaled":
            val = (val.float() * o["scale"][0]).half()
            L.nchw_to_nhwc_scaled(src, dst, o["scale"], c_off=c0)
        else:
            val = (val.float() * o["scale"][idx][:, None, None, None]).half()
            L.nchw_to_nhwc_scaled_rows(src, dst, o["scale"], c_off=c0)
        ref[..., c0:c0 + Cs] = val
        out = dst
        key = f"{tuple(src.shape)} -> {tuple(dst.shape)} c_off={c0}"
    exact = torch.equal(out, ref)
    return key, "-", 0.0 if exact else float("inf"), 0.0, {}, exact


KIND_NAMES = {0: "ddim", 1: "euler", 2: "dpmpp", 3: "ddpm"}


def _replay_cfg(sig, o, seed):
    """The CFG step kernels per sample against cfg_rescale_ddpm_ref (DDPM, phi = 0 for the plain kernel) and
    cfg_solver_ref, with the recorded coefficients; mutant: the two CFG halves swapped, and for per-row kernels the
    coefficient row of the neighbouring sample."""
    from idm_vton_b200 import lib as L
    from test_schedule_cpu import kernel_inputs
    from test_solvers_cpu import x0_prev_input
    name = sig[0]
    eps, lat = o["eps"], o["latents"]
    B, C, H, W = lat.shape
    ldc = eps.shape[-1]
    e_in, l_in, n_in = kernel_inputs(B, H, W, ldc, o["noise"] is not None, seed=seed % 1000)
    _fill(eps, e_in.to(DEV)); _fill(lat, l_in.to(DEV))
    if o["noise"] is not None:
        _fill(o["noise"], n_in.to(DEV))
    x0p = o.get("x0_prev")
    if x0p is not None:
        _fill(x0p, x0_prev_input(B, H, W, seed % 1000).to(DEV))
    coef = o["coef"].cpu()
    kinds = o["kinds"].tolist() if o.get("kinds") is not None else None
    snap = dict(eps=eps.cpu(), lat=lat.cpu(), noise=o["noise"].cpu() if o["noise"] is not None else None,
                x0=x0p.cpu() if x0p is not None else None)
    fn = getattr(L, name)
    kw = dict(do_cfg=o["do_cfg"], out=o["out"])
    if name in ("cfg_solver_step", "cfg_solver_step_rows"):
        kw.update(kind=o["kind"], x0_prev=x0p)
    if name == "cfg_step_mixed_rows":
        kw.update(kinds=o["kinds"], x0_prev=x0p)
    out = fn(eps, lat, o["noise"], o["coef"], **kw).cpu()
    assert o["do_cfg"], "the inventory's runs use CFG"
    rows = coef.dim() == 2

    def ref(b, row, swap=False):
        e = snap["eps"]
        u, t = e[b:b + 1], e[B + b:B + b + 1]
        ee = torch.cat([t, u] if swap else [u, t])
        lt = snap["lat"][b:b + 1]
        nz = snap["noise"][b:b + 1] if snap["noise"] is not None else None
        c = coef[row] if rows else coef
        kind = KIND_NAMES[kinds[b]] if kinds is not None else ("ddpm" if "ddpm" in name else o["kind"])
        if kind == "ddpm":
            phi = float(c[6]) if (name == "cfg_rescale_ddpm_step" or kinds is not None) else 0.0
            return cfg_rescale_ddpm_ref(ee, lt, nz, c[:6].tolist(), phi)
        x0 = snap["x0"][b:b + 1] if snap["x0"] is not None else None
        return cfg_solver_ref(ee, lt, nz if kind == "ddim" else None, x0, c[:8].tolist(), kind)[0]
    errs, merrs = [], collections.defaultdict(lambda: float("inf"))
    for b in range(B):
        t = ref(b, b)
        errs.append(rel_err(out[b:b + 1], t))
        merrs["CFG halves swapped"] = min(merrs["CFG halves swapped"], rel_err(ref(b, b, swap=True), t))
        if rows and B > 1 and not torch.equal(coef[b], coef[(b + 1) % B]):
            merrs["neighbour's coefficient row"] = min(merrs["neighbour's coefficient row"],
                                                       rel_err(ref(b, (b + 1) % B), t))
    return f"B={B} {H}x{W} ldc={ldc} kinds={kinds or o.get('kind', 'ddpm')}", "-", max(errs), TOL, dict(merrs), None


REPLAY = {
    "gemm": _replay_gemm, "gemm_e4m3": _replay_gemm_e4m3, "conv3x3": _replay_conv,
    "attention": lambda s, o, seed: _attn_core(o, seed, "attention"),
    "attention_rows": lambda s, o, seed: _attn_core(o, seed, "attention_rows"),
    "attention_kv8": lambda s, o, seed: _attn_core(o, seed, "attention_kv8"),
    "cross_attention": _replay_cross, "groupnorm": _replay_groupnorm, "layernorm": _replay_layernorm,
    "layernorm_e4m3": lambda s, o, seed: _replay_layernorm(s, o, seed, e4m3=True),
    "quantize_kv_e4m3": _replay_quantize_kv, "skinny_linear": _replay_skinny, "timestep_embedding": _replay_timestep,
    "upsample2x": _replay_layout, "upsample_nearest": _replay_layout, "nchw_to_nhwc": _replay_layout,
    "nchw_to_nhwc_scaled": _replay_layout, "nchw_to_nhwc_scaled_rows": _replay_layout, "nhwc_to_nchw": _replay_layout,
    "cfg_ddpm_step": _replay_cfg, "cfg_rescale_ddpm_step": _replay_cfg, "cfg_solver_step": _replay_cfg,
    "cfg_ddpm_step_rows": _replay_cfg, "cfg_solver_step_rows": _replay_cfg, "cfg_step_mixed_rows": _replay_cfg,
}
BIT_EXACT = {"conv3x3", "quantize_kv_e4m3", "upsample2x", "upsample_nearest", "nchw_to_nhwc", "nchw_to_nhwc_scaled",
             "nchw_to_nhwc_scaled_rows", "nhwc_to_nchw"}
# mutants whose distance is printed but not gated: one zero token more or less among N1 >= 768 moves the output by at
# most ~1 / N1 of its scale, below TOL_ATTN (the edge suite gates n1 +- 1 at N1 <= 128, tests/test_kernel_edges_gpu.py)
SHOWN_ONLY = ("n1-1 (shown only)",)


def _replay_one(sig):
    o = LI.build_operands(sig, DEV)
    with torch.no_grad():
        return REPLAY[sig[0]](sig, o, LI.seed_of(sig))


@pytest.fixture(scope="module")
def replayed(inventory):
    t0 = time.time()
    unique = {}
    for run, sigs in inventory["runs"].items():
        for s in sigs:
            unique.setdefault(s, run)
    results, failures = {}, []
    for sig, run in unique.items():
        key, bn, err, gate, merrs, exact = _replay_one(sig)
        torch.cuda.empty_cache()
        gated = {k: v for k, v in merrs.items() if k not in SHOWN_ONLY and v != float("inf")}
        ratio = max((err / v if v > 0 else float("inf") for v in gated.values()), default=0.0) if err > 0 else 0.0
        ok = err <= gate and (not gated or err <= 0.25 * min(gated.values()))
        if sig[0] == "gemm":
            ok = ok and (gate > 0 or exact)
        if exact is False and sig[0] in ("attention_kv8", "layernorm_e4m3", "cross_attention"):
            ok = False
        mtxt = " ".join(f"[{k}: {v:.2e}]" for k, v in merrs.items() if v != float("inf"))
        print(f"[inventory] {run:>14} {sig[0]:<24} {key:<70} bn={bn!s:<5} err={err:.3e} gate={gate:.2e} "
              f"exact={exact} mutant_ratio={ratio:.3f} {mtxt}")
        results[sig] = (run, key, err, gate, merrs, exact, ok)
        if not ok:
            failures.append(f"run {run} {sig[0]} {key}: err {err:.3e} gate {gate:.2e} exact={exact} mutants {merrs}")
    print(f"[inventory] {len(unique)} unique signatures replayed in {time.time() - t0:.1f} s")
    return dict(results=results, failures=failures)


# ------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------
def test_every_launch_matches_float64(replayed):
    assert not replayed["failures"], "launches off their float64 restatement:\n" + "\n".join(replayed["failures"])


def _families(sigs, run_a):
    fam = collections.defaultdict(int)
    mnk_a = set()
    for s in sigs:
        a = LI.args_of(s)
        n = s[0]
        if n == "gemm":
            M, K = a["a"][1]
            N = a["w"][1][0]
            fam["gemm with bias"] += a["bias"] is not None
            fam["gemm with residual"] += a["residual"] is not None
            fam["gemm GEGLU"] += bool(a["geglu"])
            if s in run_a and a["force_bn"] == 0:
                mnk_a.add((M, N, K))
        elif n == "conv3x3":
            fam["conv stride 2"] += a["stride"] == 2
            fam["conv with temb"] += a["temb"] is not None
            fam["conv two-source shortcut"] += a["sc1"] is not None
            fam["conv with residual"] += a["residual"] is not None
        elif n == "groupnorm" and a["x1"] is not None:
            C0, C1 = a["x0"][1][-1], a["x1"][1][-1]
            fam["groupnorm with x1"] += 1
            if LI.gn_groups(C0, C1)[1] is None:
                fam["groupnorm x1, no straddling group"] += 1
            else:
                fam["groupnorm x1, straddling group"] += 1
        elif n in ("attention", "attention_kv8", "attention_rows"):
            fam["attention kv1_mod"] += bool(a.get("kv1_mod"))
            fam["attention kv1_base"] += a.get("kv1_base") is not None
            fam["attention kv1_off > 0"] += a["kv1_off"] > 0
            rows = a.get("kv1_rows")
            fam["attention kv1_rows with -1"] += rows is not None and -1 in rows[6]
        elif n == "cross_attention":
            fam["cross-attention Ni = 16"] += a["ki"] is not None and a["ki"][1][1] == 16
        if n in ("gemm_e4m3", "layernorm_e4m3", "quantize_kv_e4m3", "attention_kv8"):
            fam[n] += 1
    return fam, mnk_a


REQUIRED = ("gemm with bias", "gemm with residual", "gemm GEGLU", "conv stride 2", "conv with temb",
            "conv two-source shortcut", "conv with residual", "groupnorm with x1", "groupnorm x1, straddling group",
            "groupnorm x1, no straddling group", "attention kv1_mod", "attention kv1_base", "attention kv1_off > 0",
            "attention kv1_rows with -1", "cross-attention Ni = 16", "gemm_e4m3", "layernorm_e4m3", "quantize_kv_e4m3",
            "attention_kv8")


def test_inventory_coverage(inventory, replayed):
    """The inventory is not thin: every family a full-size step must exercise is present (and was replayed above), and
    every distinct (M, N, K) of run (a) ran with the library's own tile width (force_bn = 0)."""
    allsigs = set(replayed["results"])
    fam, mnk_a = _families(allsigs, set(inventory["runs"]["a"]))
    for f in REQUIRED:
        print(f"[inventory] coverage {f:<36} {'present' if fam.get(f) else 'MISSING'} ({fam.get(f, 0)} signatures)")
    missing = [f for f in REQUIRED if not fam.get(f)]
    assert not missing, f"the launch inventory lacks {missing}"
    print(f"[inventory] run (a): {len(mnk_a)} distinct GEMM (M, N, K) at force_bn = 0: "
          + ", ".join(f"{m}x{n}x{k}->bn{LI.pick_bn(n, m, False, 0)}" for m, n, k in sorted(mnk_a)))
    assert len(mnk_a) >= 10


def test_engine_passes_what_its_state_implies(inventory):
    """The scalars the engine passes for the hoisted garment K/V: kv1_mod = the garments of the run and kv1_base a whole
    step of them inside the K/V tensor; every GEGLU weight packed for the tile width it runs at."""
    bad = []
    for run, sigs in inventory["runs"].items():
        Bg = inventory["notes"].get(run, {}).get("Bg")
        for s in sigs:
            a = LI.args_of(s)
            if s[0] in ("attention", "attention_kv8") and a.get("kv1_base") is not None:
                base = a["kv1_base"][6][0]
                B1 = (a["k1"] if s[0] == "attention" else a["kv1"][1])[1][0]
                if a["kv1_mod"] != Bg or base % Bg or base + Bg > B1:
                    bad.append(f"run {run} {s[0]}: kv1_mod {a['kv1_mod']} base {base} B1 {B1} (garments {Bg})")
            if s[0] in ("gemm", "gemm_e4m3") and a["geglu"] and a.get("pack_bn") != a["force_bn"] % 1000:
                bad.append(f"run {run} {s[0]} GEGLU: packed for bn={a.get('pack_bn')}, launched at {a['force_bn']}")
    assert not bad, "\n".join(bad)


def test_grid_operands_exact_at_the_inventory_max_k(replayed):
    """The premise of the bit-exact GEMM / convolution gates at the largest K the inventory launches (9 Cin for a
    convolution, plus the fused shortcut's channels, which accumulate separately)."""
    from test_kernel_edges_gpu import grid_sums_exact
    kmax = 0
    for s in replayed["results"]:
        a = LI.args_of(s)
        if s[0] == "gemm":
            kmax = max(kmax, a["a"][1][1])
        elif s[0] == "conv3x3":
            kmax = max(kmax, 9 * a["x"][1][-1])
    grid_sums_exact(kmax)
    print(f"[inventory] largest K {kmax}: grid operands accumulate exactly in fp32")
