"""Reference-equivalent PyTorch-eager timing on the GPU (context for BASELINE.md; not part of the product).

Runs the oracle restatement of the reference's denoiser forward (same op sequence as the reference's modules:
nn.Linear-equivalent matmuls, F.layer_norm, RMSNorm, RoPE, F.scaled_dot_product_attention, GELU) on CUDA under
`torch.autocast(bf16)` — the reference's own GPU recipe (pipeline.py:671) — at the default window shape, plus the
CFG combine / Euler update in plain torch.  This is what the hand-written kernels have to beat.
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from oracle import denoiser_oracle as do  # noqa: E402

dev = "cuda"
cfg = do.DenoiserConfig()
g = torch.Generator(device=dev).manual_seed(1234)
D, C, Dc, F_ = cfg.width, cfg.in_channels, cfg.cross_attention_dim, int(cfg.width * cfg.mlp_ratio)


def lin(o, i, bias=True):
    b = 1.0 / i ** 0.5
    w = (torch.rand(o, i, generator=g, device=dev) * 2 - 1) * b
    return w, ((torch.rand(o, generator=g, device=dev) * 2 - 1) * b if bias else None)


sd = {}
sd["proj_in.weight"], sd["proj_in.bias"] = lin(D, C)
sd["time_proj.linear_1.weight"], sd["time_proj.linear_1.bias"] = lin(4 * D, D)
sd["time_proj.linear_2.weight"], sd["time_proj.linear_2.bias"] = lin(D, 4 * D)
sd["norm_out.weight"], sd["norm_out.bias"] = torch.ones(D, device=dev), torch.zeros(D, device=dev)
sd["proj_out.weight"], sd["proj_out.bias"] = lin(C, D)
for i in range(cfg.num_layers):
    p = f"blocks.{i}."
    if i > cfg.num_layers // 2:
        sd[p + "linear_skip.weight"], sd[p + "linear_skip.bias"] = lin(D, 2 * D)
        sd[p + "norm_skip.weight"], sd[p + "norm_skip.bias"] = torch.ones(D, device=dev), torch.zeros(D, device=dev)
    for n in ("norm_s_attn", "norm_x_attn", "norm_ff"):
        sd[p + n + ".weight"], sd[p + n + ".bias"] = torch.ones(D, device=dev), torch.zeros(D, device=dev)
    for a, kd in (("s_attn", D), ("x_attn", Dc)):
        sd[p + a + ".to_q.weight"], _ = lin(D, D, False)
        sd[p + a + ".to_k.weight"], _ = lin(D, kd, False)
        sd[p + a + ".to_v.weight"], _ = lin(D, kd, False)
        sd[p + a + ".norm_q.weight"] = torch.ones(128, device=dev)
        sd[p + a + ".norm_k.weight"] = torch.ones(128, device=dev)
        sd[p + a + ".to_out.0.weight"], sd[p + a + ".to_out.0.bias"] = lin(D, D)
    sd[p + "ff.net.0.proj.weight"], sd[p + "ff.net.0.proj.bias"] = lin(F_, D)
    sd[p + "ff.net.2.weight"], sd[p + "ff.net.2.bias"] = lin(D, F_)

# the oracle helpers build a few constants on the CPU; patch them onto the device for this timing run
_te, _rt = do.timestep_embedding, do.rotary_tables
do.timestep_embedding = lambda t, c: _te(t.cpu(), c).to(dev)
do.rotary_tables = lambda hd, pos: tuple(x.to(dev) for x in _rt(hd, pos.cpu()))

T, N = 16, 2048
lat = torch.randn(1, T, N, C, device=dev)
ctx = torch.randn(1, T, 257, Dc, device=dev)
mask = torch.zeros(1, T, device=dev)
mask[0, 0] = 1
fs = torch.arange(T, dtype=torch.float32, device=dev)[None]


def step(freqs):
    h, c, m, f = do.cfg_batch(lat, ctx, mask, fs, ((0, 1), (1, 1)))
    t = torch.tensor([500.0, 500.0], device=dev)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out, freqs = do.denoiser_forward(sd, cfg, h, c, f, t, m, freqs)
    v = do.cfg_aggregate(out, [7.5], 2)
    upd = lat + 0.01 * v
    lat[mask == 0] = upd[mask == 0].float()
    return freqs


with torch.no_grad():
    fr = step(None)
    fr = step(fr)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        fr = step(fr)
    e1.record()
    torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / 3
print(f"REF_GPU_EAGER ms_per_step {ms:.1f} steps_per_s {1000.0 / ms:.3f} model_TFLOPs {5.469e14 / ms / 1e9:.0f} "
      f"(torch {torch.__version__}, autocast bf16, SDPA backend default)")
