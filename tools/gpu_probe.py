"""Kernel bring-up probe (runs on the GPU box).  Each group runs in its own subprocess so a trapped kernel cannot
poison the CUDA context of the next group.  Results -> <temp dir>/actionmesh_b200_probe/probe_<group>.json + stdout summary.

    python tools/gpu_probe.py            # all groups
    python tools/gpu_probe.py gemm attn  # selected groups
"""
from __future__ import annotations

import json
import math
import os
import subprocess
import sys
import tempfile
import time
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(tempfile.gettempdir(), "actionmesh_b200_probe")


def _err(a, b):
    import torch
    a = a.float()
    b = b.float()
    d = (a - b).abs()
    return {"max_abs": float(d.max()), "mean_abs": float(d.mean()), "ref_absmax": float(b.abs().max()),
            "rel_fro": float(d.norm() / (b.norm() + 1e-30)), "nan": bool(torch.isnan(a).any())}


def _time(fn, iters=5, warm=2):
    import torch
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True)
    e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def group_elementwise(res):
    import torch
    from actionmesh_b200 import ops
    dev = "cuda"
    g = torch.Generator(device="cpu").manual_seed(0)
    # --- K9
    T, NPF = 16, 2048 * 64
    lat = torch.randn(1, T, 2048, 64, generator=g).to(dev)
    pred_full = torch.randn(2, T, 2049, 64, generator=g).to(dev).bfloat16()
    upd = torch.ones(T, dtype=torch.uint8)
    upd[0] = 0
    upd[7] = 0
    upd = upd.to(dev)
    ref = lat.clone()
    p = pred_full[:, :, 1:, :].float()
    v = p[0] + 7.5 * (p[1] - p[0])
    dt = 0.0113
    refu = ref + dt * v[None]
    mask = upd.bool()
    ref[0, mask] = refu[0, mask]
    x = lat.clone()
    ops.cfg_euler_step(x, pred_full, [7.5], dt, upd, n_branches=2, branch_stride=T * 2049 * 64,
                       frame_stride=2049 * 64, frame_offset=64, n_per_frame=NPF)
    torch.cuda.synchronize()
    res["k9"] = _err(x, ref)
    res["k9"]["observed_bit_identical"] = bool(torch.equal(x[0, 0], lat[0, 0]) and torch.equal(x[0, 7], lat[0, 7]))
    ms = _time(lambda: ops.cfg_euler_step(x, pred_full, [7.5], dt, upd, n_branches=2, branch_stride=T * 2049 * 64,
                                          frame_stride=2049 * 64, frame_offset=64, n_per_frame=NPF), iters=20)
    nb = int(mask.sum()) * NPF * 12
    res["k9"]["ms"] = ms
    res["k9"]["GBps"] = nb / ms / 1e6
    # --- layernorm
    for cols in (1024, 2048):
        for dt_ in (torch.bfloat16, torch.float32):
            xx = (torch.randn(1000, cols, generator=g) * 2 + 0.5).to(dev).to(dt_)
            gm = torch.randn(cols, generator=g).to(dev)
            bt = torch.randn(cols, generator=g).to(dev)
            y = ops.layernorm(xx, gm, bt, 1e-5)
            r = torch.nn.functional.layer_norm(xx.float(), (cols,), gm, bt, 1e-5)
            res[f"ln_{cols}_{str(dt_)[6:]}"] = _err(y, r)
    xx = torch.randn(65568, 2048, generator=g).to(dev).bfloat16()
    gm = torch.ones(2048, device=dev)
    bt = torch.zeros(2048, device=dev)
    out = torch.empty_like(xx)
    ms = _time(lambda: ops.layernorm(xx, gm, bt, 1e-5, out=out), iters=10)
    res["ln_big"] = {"ms": ms, "GBps": xx.numel() * 4 / ms / 1e6}
    # --- cast / timestep / bias rows
    a = torch.randn(4099, generator=g).to(dev)
    res["cast"] = _err(ops.cast_bf16(a), a.bfloat16())
    t = torch.tensor([0.0, 8.9285717, 502.98, 1000.0], device=dev)
    emb = ops.timestep_embedding(t, 2048)
    half = 1024
    w = torch.exp(-math.log(10000.0) * torch.arange(half, device=dev, dtype=torch.float32) / half)
    e = t[:, None] * w[None]
    res["timestep_emb"] = _err(emb, torch.cat([e.sin(), e.cos()], -1))
    y = torch.randn(100, 2048, generator=g).to(dev).bfloat16()
    b = torch.randn(2048, generator=g).to(dev)
    r = (y.float() + b).bfloat16()
    ops.add_bias_rows(y, b)
    res["add_bias_rows"] = _err(y, r)


def _gemm_kernel(fn):
    """Name of the GEMM kernel one call of fn launches (gemm_bf16_kernel<BN>), read from a torch.profiler trace."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    names = set()
    for _ in range(3):  # a short trace now and then comes back without its kernel record
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if "gemm_bf16_kernel" in e.name}
        if names:
            break
    return ",".join(sorted(n[n.index("gemm_bf16_kernel"):].split("(")[0] for n in names))


def _gemm_case(res, name, m, n, k, *, bias=False, act=0, residual=False, a2=False, row_map=None, out_fp32=False,
               res_fp32=False, col_scale=False, norm=None, timing=False, seed=1, alias=False, out2=False):
    import torch
    from actionmesh_b200 import ops
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(seed)
    A = (torch.randn(m, k, generator=g, device=dev) * 0.5).bfloat16()
    W = (torch.randn(n, k, generator=g, device=dev) / math.sqrt(k)).bfloat16()
    kw = {}
    ref = A.float() @ W.float().t()
    if a2:
        k1 = k // 2
        A1 = A[:, :k1].contiguous()
        A2 = A[:, k1:].contiguous()
        kw["a2"] = A2
        Ain = A1
    else:
        Ain = A
    if norm is not None:
        nc, seg, rc, rpp = norm
        w0 = torch.rand(128, generator=g, device=dev) + 0.5
        w1 = torch.rand(128, generator=g, device=dev) + 0.5
        npos = (m + rpp - 1) // rpp
        ang = torch.rand(npos, 64, generator=g, device=dev) * 6.28
        cos, sin = ang.cos(), ang.sin()
        kw["norm"] = dict(cols=nc, seg=seg, w0=w0, w1=w1, eps=1e-6, rope_cols=rc, cos=cos, sin=sin, rows_per_pos=rpp)
        r = ref.clone()
        for c0 in range(0, nc, 128):
            h = r[:, c0:c0 + 128]
            h = h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + 1e-6) * (w0 if c0 < seg else w1)
            if c0 < rc:
                pos = torch.arange(m, device=dev) // rpp
                cc = cos[pos].repeat_interleave(2, dim=1)
                ss = sin[pos].repeat_interleave(2, dim=1)
                x0, x1 = h.reshape(m, 64, 2).unbind(-1)
                rot = torch.stack([-x1, x0], -1).reshape(m, 128)
                h = h * cc + rot * ss
            r[:, c0:c0 + 128] = h
        ref = r
    if bias:
        bv = torch.randn(n, generator=g, device=dev)
        kw["bias"] = bv
        if norm is None:
            ref = ref + bv
        else:
            ref[:, norm[0]:] += bv[norm[0]:]
    if act:
        kw["act"] = 1
        ref = torch.nn.functional.gelu(ref)
    if col_scale:
        cs = torch.randn(n, generator=g, device=dev)
        kw["col_scale"] = cs
        ref = ref * cs
    mo = m
    if row_map is not None:
        gr, gs, ro = row_map
        mo = (m // gr) * gs + ro + gr
        kw["row_map"] = row_map
    out = torch.full((mo, n), 7.0, device=dev, dtype=torch.float32 if out_fp32 else torch.bfloat16)
    if residual:
        R = torch.randn(mo, n, generator=g, device=dev)
        R = R if res_fp32 else R.bfloat16()
        if alias:  # the residual stream updated in place, as the denoiser runs it
            out.copy_(R)
            kw["residual"] = out
        else:
            kw["residual"] = R
    if out2:
        kw["out2"] = torch.empty(mo, n, device=dev, dtype=torch.bfloat16)
    ops.gemm(Ain, W, out, **kw)
    torch.cuda.synchronize()
    if row_map is not None:
        gr, gs, ro = row_map
        rows = torch.arange(m, device=dev)
        drow = (rows // gr) * gs + rows % gr + ro
        full = torch.full((mo, n), 7.0, device=dev)
        if residual:
            full[drow] = ref + R.float()[drow]
        else:
            full[drow] = ref
        ref = full
    elif residual:
        ref = ref + R.float()
    res[name] = _err(out, ref)
    if timing:
        ms = _time(lambda: ops.gemm(Ain, W, out, **kw), iters=20)
        res[name]["ms"] = ms
        res[name]["TFLOPs"] = 2.0 * m * n * k / ms / 1e9
        res[name]["kernel"] = _gemm_kernel(lambda: ops.gemm(Ain, W, out, **kw))


def group_gemm(res):
    _gemm_case(res, "g_basic_128x256x64", 128, 256, 64)
    _gemm_case(res, "g_256x256x128", 256, 256, 128)
    _gemm_case(res, "g_n128_tail_m300", 300, 128, 192)
    _gemm_case(res, "g_n64", 200, 64, 128, bias=True, out_fp32=True)
    _gemm_case(res, "g_multi_tile_persist", 128 * 40, 2048, 256)   # > 132 tiles => more than one wave of CTAs
    _gemm_case(res, "g_bias_gelu_res", 512, 512, 256, bias=True, act=1, residual=True)
    _gemm_case(res, "g_a2_split", 384, 256, 512, a2=True, bias=True)
    _gemm_case(res, "g_rowmap", 256, 256, 64, bias=True, row_map=(64, 65, 1))
    _gemm_case(res, "g_fp32_res_colscale", 257, 256, 128, bias=True, residual=True, res_fp32=True, out_fp32=True, col_scale=True)
    _gemm_case(res, "g_norm_rope_qkv", 300, 768, 256, norm=(512, 256, 512, 100))
    _gemm_case(res, "g_norm_only_q", 300, 256, 256, norm=(256, 256, 0, 1))
    _gemm_case(res, "g_norm_kv_bias", 300, 512, 128, norm=(256, 256, 0, 1), bias=True)


def _cublas_case(res, m, n, k):
    """torch.matmul (cuBLAS) on the same bf16 shape, bf16 out and no epilogue: a measured ceiling beside our number."""
    import torch
    a = torch.randn(m, k, device="cuda").bfloat16()
    w = torch.randn(n, k, device="cuda").bfloat16()
    ms = _time(lambda: torch.matmul(a, w.t()), iters=5)
    res[f"cublas_{m}x{n}x{k}"] = {"ms": ms, "TFLOPs": 2.0 * m * n * k / ms / 1e9}


def group_gemm_perf(res):
    res["card"] = _card()
    _gemm_case(res, "p_8192x2048x2048", 8192, 2048, 2048, timing=True)
    _gemm_case(res, "p_65568x2048x2048_res", 65568, 2048, 2048, bias=True, residual=True, timing=True)
    _gemm_case(res, "p_65568x8192x2048_gelu", 65568, 8192, 2048, bias=True, act=1, timing=True)
    _gemm_case(res, "p_65568x2048x8192_res", 65568, 2048, 8192, bias=True, residual=True, timing=True)
    _gemm_case(res, "p_65568x6144x2048_qkv", 65568, 6144, 2048, norm=(4096, 2048, 4096, 2049), timing=True)
    _gemm_case(res, "p_65568x2048x4096_skip", 65568, 2048, 4096, a2=True, bias=True, timing=True)
    # the block GEMMs with the epilogues the fp32-stream denoiser launches: s.o and x.o update the fp32 residual stream in
    # place, ff2 also writes its bf16 copy; x.q (q-norm) and x.o run once per CFG branch with image context (M = 16 x 2049)
    _gemm_case(res, "p_65568x2048x2048_s.o_f32", 65568, 2048, 2048, bias=True, residual=True, res_fp32=True, out_fp32=True,
               alias=True, timing=True)
    _gemm_case(res, "p_65568x2048x8192_ff2_f32", 65568, 2048, 8192, bias=True, residual=True, res_fp32=True, out_fp32=True,
               alias=True, out2=True, timing=True)
    _gemm_case(res, "p_32784x2048x2048_x.q", 32784, 2048, 2048, norm=(2048, 2048, 0, 1), timing=True)
    _gemm_case(res, "p_32784x2048x2048_x.o_f32", 32784, 2048, 2048, bias=True, residual=True, res_fp32=True, out_fp32=True,
               alias=True, timing=True)
    for m, n, k in ((8192, 2048, 2048), (65568, 2048, 2048), (65568, 8192, 2048), (65568, 2048, 8192),
                    (65568, 6144, 2048), (65568, 2048, 4096), (32784, 2048, 2048)):
        _cublas_case(res, m, n, k)


def _attn_ref(q, k, v, scale):
    import torch
    # q:(B,Sq,H,D)
    qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))
    s = (qf @ kf.transpose(-1, -2)) * scale
    p = s.softmax(-1)
    return (p @ vf).permute(0, 2, 1, 3)


def _attn_case(res, name, B, H, Sq, Sk, D, *, mode="rand", fused=False, timing=False, seed=3, kv_chunks=1):
    import torch
    from actionmesh_b200 import ops
    dev = "cuda"
    g = torch.Generator(device="cpu").manual_seed(seed)
    scale = 1.0 / math.sqrt(D)
    if fused:
        assert Sq == Sk
        buf = torch.randn(B, Sq, 3 * H * D, generator=g).to(dev).bfloat16()
        q = buf[:, :, 0 * H * D:1 * H * D].view(B, Sq, H, D)
        k = buf[:, :, 1 * H * D:2 * H * D].view(B, Sq, H, D)
        v = buf[:, :, 2 * H * D:3 * H * D].view(B, Sq, H, D)
    else:
        q = torch.randn(B, Sq, H, D, generator=g).to(dev).bfloat16()
        k = torch.randn(B, Sk, H, D, generator=g).to(dev).bfloat16()
        v = torch.randn(B, Sk, H, D, generator=g).to(dev).bfloat16()
    if mode == "vones":
        v = torch.ones_like(v)
    elif mode == "kzero":
        k = torch.zeros_like(k)
    elif mode == "sharp":
        q = q * 4
    elif mode == "spike":  # ONE key (tile 10, column 3: a slot whose exponential runs on the FMA pipe for half of the rows) scores
        u = torch.zeros(D, device=dev)  # 75-225 nats above everything else: exp2 arguments far past 127 in the fast pass
        u[0] = 1.0
        q = (q.float() + 4.0 * u).bfloat16()
        k = k.clone()
        k[:, 128 * 10 + 3] = (424.0 * u).bfloat16()
    elif mode == "sharp8":  # logits with std 8: most rows leave the fixed-reference safe range after the first key tile
        q = q * 8
    out = torch.full((B, Sq, H, D), 3.0, device=dev, dtype=torch.bfloat16)
    if kv_chunks > 1:
        kc = k.view(B, kv_chunks, Sk // kv_chunks, H, D)
        vc = v.view(B, kv_chunks, Sk // kv_chunks, H, D)
        ops.flash_attn(q, kc, vc, out, scale, kv_chunks=kv_chunks)
    else:
        ops.flash_attn(q, k, v, out, scale)
    torch.cuda.synchronize()
    if Sq * Sk * B * H <= 2 ** 31:
        ref = _attn_ref(q, k, v, scale)
    else:
        ref = torch.nn.functional.scaled_dot_product_attention(
            q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), v.permute(0, 2, 1, 3)).permute(0, 2, 1, 3)
    res[name] = _err(out, ref)
    if timing:
        if kv_chunks > 1:
            fn = lambda: ops.flash_attn(q, kc, vc, out, scale, kv_chunks=kv_chunks)
        else:
            fn = lambda: ops.flash_attn(q, k, v, out, scale)
        ms = _time(fn, iters=3, warm=1)
        res[name]["ms"] = ms
        res[name]["TFLOPs"] = 4.0 * B * H * Sq * Sk * D / ms / 1e9


def group_attn(res):
    _attn_case(res, "a_1tile_vones", 1, 1, 256, 64, 128, mode="vones")
    _attn_case(res, "a_1tile_kzero", 1, 1, 256, 64, 128, mode="kzero")
    _attn_case(res, "a_1tile_rand", 1, 1, 256, 64, 128)
    _attn_case(res, "a_2tiles", 1, 1, 256, 128, 128)
    _attn_case(res, "a_5tiles_stagewrap", 1, 2, 256, 320, 128)
    _attn_case(res, "a_tails_q300_k257", 2, 2, 300, 257, 128)
    _attn_case(res, "a_sharp_rescale", 1, 2, 512, 1024, 128, mode="sharp")
    _attn_case(res, "a_fused_qkv_strided", 2, 4, 520, 520, 128, fused=True)
    _attn_case(res, "a_chunks2", 2, 2, 256, 2 * 200, 128, kv_chunks=2)
    _attn_case(res, "a_d64_s257", 3, 4, 257, 257, 64)
    _attn_case(res, "a_d64_fused", 2, 16, 257, 257, 64, fused=True)


def group_attn_perf(res):
    _attn_case(res, "ap_s4098", 1, 16, 4098, 4098, 128, timing=True)
    _attn_case(res, "ap_cross_2049x257", 16, 16, 2049, 257, 128, timing=True)
    _attn_case(res, "ap_s32784_full", 2, 16, 32784, 32784, 128, fused=True, timing=True)
    import torch
    q = torch.randn(2, 16, 32784, 128, device="cuda").bfloat16()
    ms = _time(lambda: torch.nn.functional.scaled_dot_product_attention(q, q, q), iters=2, warm=1)
    res["torch_sdpa_s32784"] = {"ms": ms, "TFLOPs": 4.0 * 2 * 16 * 32784 * 32784 * 128 / ms / 1e9}


def group_attn_more(res):
    """Shapes of the frame-sharded window, ragged chunks, a growing row maximum (slow path after the first tile)."""
    import torch
    from actionmesh_b200 import ops
    _attn_case(res, "am_single", 1, 1, 1, 1, 128)
    _attn_case(res, "am_q129_k129", 1, 3, 129, 129, 128)
    _attn_case(res, "am_3tiles_tail1", 2, 2, 700, 257, 128)
    _attn_case(res, "am_12tiles", 1, 2, 384, 1536, 128)
    _attn_case(res, "am_chunks8", 1, 2, 2 * 2049, 8 * 2 * 2049, 128, kv_chunks=8)
    _attn_case(res, "am_chunks8_64keys", 1, 2, 64, 8 * 64, 128, kv_chunks=8)       # every tile is a ragged tail tile
    _attn_case(res, "am_chunks4_200keys", 2, 2, 300, 4 * 200, 128, kv_chunks=4)
    _attn_case(res, "am_window_t2", 2, 16, 2 * 2049, 2 * 2049, 128, fused=True)
    _attn_case(res, "am_sharp16", 1, 2, 512, 2048, 128, mode="sharp")
    g = torch.Generator().manual_seed(5)
    B, S, H, D = 1, 128 * 9 + 17, 2, 128
    q = torch.randn(B, S, H, D, generator=g)
    k = torch.randn(B, S, H, D, generator=g) * 0.05
    v = torch.randn(B, S, H, D, generator=g)
    qdir = q.mean(dim=1, keepdim=True)
    qdir = qdir / qdir.norm(dim=-1, keepdim=True)
    ramp = (torch.arange(S, dtype=torch.float32) / 128.0).floor()[None, :, None, None]
    k = k + ramp * 12.0 * qdir * (math.sqrt(D) / (q * qdir).sum(-1, keepdim=True).abs().mean())
    q, k, v = (t.cuda().bfloat16() for t in (q, k, v))
    o = torch.empty_like(q)
    ops.flash_attn(q, k, v, o, 1 / math.sqrt(D))
    res["am_late_rescale"] = _err(o, _attn_ref(q, k, v, 1 / math.sqrt(D)))


def _card():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        pl = "unknown"
    return {"name": torch.cuda.get_device_name(), "power_limit": pl}


def group_vae_decode(res):
    """TripoSG VAE decode + anchor-mesh extraction at full width (1024, 8 heads, 16 layers, 2048 latent tokens).
    TFLOP/s of the query path from the shape count: q-proj 2D^2 + attention 4 Sk D + o-proj 2D^2 + FF 16 D^2 per point."""
    import torch

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import triposg_vae_ref as ref
    from actionmesh_b200.triposg_vae import B200TripoSGVAE, mesh_from_grid, refine_octree

    res["card"] = _card()
    D, Sk = 1024, 2048
    sd = ref.make_state_dict(D, 8, 16, seed=1)
    vae = B200TripoSGVAE().to("cuda")
    vae.load_state_dict(sd)
    g = torch.Generator(device="cuda").manual_seed(0)
    z = torch.randn(2048, 64, device="cuda", generator=g)
    ctx = vae.prepare(z)
    res["trunk_kv_ms"] = {"ms": _time(lambda: vae.prepare(z), iters=5)}
    flop_pt = 2 * D * D + 4 * Sk * D + 2 * D * D + 16 * D * D
    for P in (262144, 2097152):
        pts = torch.rand(P, 3, device="cuda", generator=g) * 2.01 - 1.005
        ms = _time(lambda: vae.query(ctx, pts), iters=3, warm=1)
        res[f"query_{P}"] = {"ms": ms, "tflops": flop_pt * P / ms / 1e9}
    # the reference's recipe: fp32 modules under fp16 autocast, <= 10000 points per vae.decode call, trunk recomputed per call
    sdc = {k: v.cuda() for k, v in sd.items()}
    for P in (262144, 2097152):
        pts = torch.rand(1, P, 3, device="cuda", generator=g) * 2.01 - 1.005

        def recipe():
            with torch.autocast("cuda", dtype=torch.float16):
                for i in range(0, P, 10000):
                    ref.decode_fp32(sdc, z[None], pts[:, i:i + 10000], 8, 16)

        ms = _time(recipe, iters=1, warm=1)
        res[f"reference_recipe_{P}"] = {"ms": ms, "calls": (P + 9999) // 10000}
    t = {}

    def extract():
        grid = refine_octree(ref.sphere, ref.BOUNDS, 9)
        torch.cuda.synchronize()
        t["refine"] = time.time()
        v, f = mesh_from_grid(grid, ref.BOUNDS, 9)
        t["nv"], t["nf"] = len(v), len(f)
        return grid

    for _ in range(2):
        torch.cuda.synchronize()
        t0 = time.time()
        grid = extract()
        t1 = time.time()
    res["sphere_depth9"] = {"refine_ms": (t["refine"] - t0) * 1e3, "dmc_ms": (t1 - t["refine"]) * 1e3,
                            "total_ms": (t1 - t0) * 1e3, "vertices": t["nv"], "faces": t["nf"],
                            "queried": int(torch.isfinite(grid).sum())}


def group_vae_encode(res):
    """TripoSG VAE encoder of the mesh-input path at full width (512, 8 heads x 64, 8 layers; 16384 surface points -> 2048
    tokens): the FPS kernel (8192 -> 2048), the encoder launch program, the whole encode_to_latent, and the reference's recipe
    (the fp32 restatement under fp16 autocast).  pytorch3d's FPS, which the reference uses, is not installed and not timed.
    FLOPs: proj_in 2 (T + N) 64 W, cross q/o 4 T W^2, cross K/V 4 N W^2, FF 16 T W^2 per block, self QKV/o 8 T W^2,
    attention 4 T N W (cross) and 4 T^2 W (self), quant 2 T W 128."""
    import torch

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import triposg_vae_encoder_ref as ref
    import triposg_vae_ref as dref
    from actionmesh_b200 import ops
    from actionmesh_b200.triposg_vae import B200TripoSGVAE

    res["card"] = _card()
    W, L, T, N = 512, 8, 2048, 16384
    sd = dref.make_state_dict(1024, 8, 1, seed=1)
    enc = ref.make_encoder_state_dict(W, 8, L, seed=2)
    sd.update(enc)
    vae = B200TripoSGVAE(num_layers_decoder=1).to("cuda")
    vae.load_state_dict(sd)
    surface = ref.sphere_surface(N, 3).cuda()
    sub = surface[:, :4 * T].contiguous()
    start = torch.tensor([17], device="cuda")
    res["fps_8192_2048"] = {"ms": _time(lambda: ops.farthest_point_sample(sub, T, start), iters=20, warm=3)}
    sampled, _ = vae.sample_features(surface, T, seed=0, generator=torch.Generator().manual_seed(0))
    attn = 4 * T * N * W + L * 4 * T * T * W
    flop = 2 * (T + N) * 64 * W + 4 * T * W * W + 4 * N * W * W + (L + 1) * 16 * T * W * W + L * 8 * T * W * W + attn \
        + 2 * T * W * 128
    ms = _time(lambda: vae.encode_points(surface[0], sampled[0]), iters=10, warm=2)
    res["encoder_program"] = {"ms": ms, "tflops": flop / ms / 1e9, "gflop": flop / 1e9, "attn_gflop": attn / 1e9}
    res["encode_to_latent"] = {"ms": _time(lambda: vae.encode_to_latent(surface, seed=0, generator=torch.Generator().manual_seed(0)),
                                           iters=10, warm=2)}
    sdc = {k: v.cuda() for k, v in enc.items()}

    def recipe():
        with torch.autocast("cuda", dtype=torch.float16):
            ref.encode_fp32(sdc, surface, sampled, 8, L)

    ms = _time(recipe, iters=5, warm=2)
    res["reference_recipe_encoder"] = {"ms": ms, "tflops": flop / ms / 1e9}


def group_mesh_process(res):
    """Anchor-mesh post-processing at Stage 0's size: depth-9 sphere and torus from refine_octree + mesh_from_grid; host clean,
    GPU decimation to 40 000 faces (with its round count) and floater removal (threshold 0.02), each timed with a host clock
    around synchronised calls (second of two runs).  Then the Stage-II vertex-query block (full-width random weights, one
    16-frame window, one target) at the undecimated and the decimated vertex count: the whole autoencoder call, and the
    CUDA-event time of the query block's GEMMs (tag s2_q).  fast_simplification is not installed and not timed."""
    import numpy as np
    import torch

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import triposg_vae_ref as ref
    from actionmesh_b200 import ops
    from actionmesh_b200.autoencoder import AutoencoderConfig, B200Autoencoder
    from actionmesh_b200.mesh_input import clean_topology
    from actionmesh_b200.mesh_process import decimate, remove_floaters
    from actionmesh_b200.triposg_vae import mesh_from_grid, refine_octree

    res["card"] = _card()
    counts = {}
    for name, field in (("sphere", ref.sphere), ("torus", ref.torus)):
        v, f = mesh_from_grid(refine_octree(field, ref.BOUNDS, 9), ref.BOUNDS, 9)
        r = {}
        for _ in range(2):
            t0 = time.time()
            v0, f0 = clean_topology(v.astype(np.float64), f.astype(np.int64))
            t1 = time.time()
            pos = torch.from_numpy(v0).cuda()
            ft = torch.from_numpy(f0.astype(np.int32)).cuda()
            work, scan = ops.mesh_scan_scratch(len(v0), len(f0), "cuda")
            torch.cuda.synchronize()
            t2 = time.time()
            pos, ft, rounds = decimate(pos, ft, 40000, work, scan)
            torch.cuda.synchronize()
            t3 = time.time()
            pos2, ft2 = remove_floaters(pos, ft, 0.02, work, scan)
            torch.cuda.synchronize()
            t4 = time.time()
            r = {"vertices_in": len(v0), "faces_in": len(f0), "clean_ms": (t1 - t0) * 1e3, "decimate_ms": (t3 - t2) * 1e3,
                 "rounds": rounds, "faces_out": int(ft.shape[0]), "vertices_out": int(pos.shape[0]),
                 "floaters_ms": (t4 - t3) * 1e3, "faces_after_floaters": int(ft2.shape[0])}
        res[f"{name}_depth9"] = r
        counts[name] = (r["vertices_in"], r["vertices_out"])
    ae = B200Autoencoder(AutoencoderConfig()).to("cuda")
    ae.init_random_(seed=3)
    g = torch.Generator().manual_seed(0)
    T, N = 16, 2048
    lat = torch.randn(1, T, N, 64, generator=g).cuda()
    fs = torch.arange(T, dtype=torch.float32)[None]
    src, tgt = torch.zeros(1), torch.full((1, 1), 0.5)
    for label, V in (("undecimated", counts["sphere"][0]), ("decimated", counts["sphere"][1])):
        q = torch.randn(1, V, 6, generator=g)
        q[..., 3:] = torch.nn.functional.normalize(q[..., 3:], dim=-1)
        q = q.cuda()
        ae(latent=lat, framestep=fs, source_alpha=src, target_alphas=tgt, query=q)
        torch.cuda.synchronize()
        ops.event_log, ops.event_tags = [], {"s2_q"}
        t0 = time.time()
        ae(latent=lat, framestep=fs, source_alpha=src, target_alphas=tgt, query=q)
        torch.cuda.synchronize()
        ms = (time.time() - t0) * 1e3
        qms = sum(e0.elapsed_time(e1) for _, e0, e1, _ in ops.event_log)
        ops.event_log, ops.event_tags = None, set()
        res[f"stage2_{label}"] = {"vertices": V, "autoencoder_call_ms": ms, "query_gemm_ms": qms}


GROUPS = {
    "elementwise": group_elementwise, "gemm": group_gemm, "attn": group_attn, "attn_more": group_attn_more,
    "gemm_perf": group_gemm_perf, "attn_perf": group_attn_perf, "vae_decode": group_vae_decode,
    "vae_encode": group_vae_encode, "mesh_process": group_mesh_process,
}
TAG = os.environ.get("AMB_PROBE_TAG", "")
if os.environ.get("AMB_PROBE_LIB"):  # bring-up only: probe an experimental build (tools/build_variant.sh) instead of the product library
    from actionmesh_b200 import _lib as _amb_lib

    _amb_lib.LIB_PATH = os.path.abspath(os.environ["AMB_PROBE_LIB"])


def run_group(name):
    import torch
    res = {}
    t0 = time.time()
    try:
        GROUPS[name](res)
        torch.cuda.synchronize()
        res["_status"] = "ok"
    except Exception as e:  # noqa: BLE001
        res["_status"] = "EXC: " + repr(e)[:400]
        res["_trace"] = traceback.format_exc()[-1500:]
    res["_sec"] = time.time() - t0
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, f"probe_{name}{TAG}.json"), "w") as f:
        json.dump(res, f, indent=1)
    return res


def main():
    args = sys.argv[1:]
    if args and args[0] == "--child":
        run_group(args[1])
        return
    names = args or list(GROUPS)
    for n in names:
        t0 = time.time()
        stale = os.path.join(OUT, f"probe_{n}{TAG}.json")
        if os.path.exists(stale):
            os.remove(stale)
        try:
            pr = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", n], capture_output=True, text=True,
                                timeout=420)
            tail = (pr.stdout + pr.stderr)[-1200:]
        except subprocess.TimeoutExpired:
            tail = "TIMEOUT"
        path = os.path.join(OUT, f"probe_{n}{TAG}.json")
        print(f"==== {n}{TAG} ({time.time() - t0:.0f}s)")
        if os.path.exists(path):
            r = json.load(open(path))
            for k, v in r.items():
                if k.startswith("_trace"):
                    continue
                if isinstance(v, dict):
                    s = " ".join(f"{a}={b:.4g}" if isinstance(b, float) else f"{a}={b}" for a, b in v.items())
                else:
                    s = str(v)
                print(f"  {k}: {s}")
            if r.get("_status") != "ok":
                print(r.get("_trace", ""))
                print("  child tail:", tail[-600:])
        else:
            print("  NO RESULT FILE; child tail:", tail)


if __name__ == "__main__":
    main()
