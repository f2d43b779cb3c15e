"""Vertex-level parity as the metric `north_star` names (-m gpu): Chamfer distance (actionbench/chamfer.py restatement)
between the per-frame vertices decoded from the CUDA path's latents and from the REFERENCE's latents (golden 4-step
CFG-7.5 trajectories produced by the reference's own SchedulerFlow + ActionMeshDenoiser in fp32), both decoded by the same
fp32 Stage-II decoder restatement so that only the Stage-I difference is measured (the CUDA Stage II has its own parity
test, tests/test_autoencoder_gpu.py).  Vertices live in [-1, 1]^3.

Eight (weight seed, input seed) draws (tests/golden/denoiser_tiny_multiseed.pt, written by oracle/gen_golden.py from the
reference's modules).  Yardstick: the reference's OWN modules under its own mixed-precision recipe (pipeline.py:671
autocast bf16) against the same fp32 trajectories — what "bf16 vs fp32" costs the reference itself.  The bar is on the
MEAN over the draws: the CUDA path's Chamfer may not exceed 1.25x the reference-autocast Chamfer, nor may its latent
error; the default fp32 residual stream is expected well below both (reported in chamfer_report.json under the system temp directory)."""
import json
import os
import tempfile

import pytest
import torch

from conftest import load_golden
from oracle import autoencoder_oracle as ao
from oracle import synth

REPORT_DIR = os.path.join(tempfile.gettempdir(), "actionmesh_b200_reports")

pytestmark = pytest.mark.gpu


def _decode_setup():
    acfg = ao.AutoencoderConfig(width=256, num_layers=2, num_attention_heads=2)
    asd = ao.make_autoencoder_state_dict(acfg, 4321)
    gen = torch.Generator().manual_seed(12)
    pts = torch.randn(1, 4000, 3, generator=gen)
    pts = pts / pts.norm(dim=-1, keepdim=True) * 0.6           # a sphere as the "anchor mesh" vertex cloud
    query = torch.cat([pts, pts / 0.6], dim=-1)                # vertices + normals (in_extra_channels = 3)
    return acfg, asd, pts, query


def _chamfer_mean(acfg, asd, pts, query, lat_a, lat_b, fs):
    sa, ta = torch.tensor([0.0]), torch.linspace(0, 1, 3)[None]
    va = ao.apply_displacement(pts, ao.autoencoder_forward(asd, acfg, lat_a, fs, sa, ta, query))
    vb = ao.apply_displacement(pts, ao.autoencoder_forward(asd, acfg, lat_b, fs, sa, ta, query))
    cds = [ao.chamfer_score(va[0, t].numpy(), vb[0, t].numpy(), n=10_000, seed=44) for t in range(3)]
    return sum(cds) / 3, cds


def test_chamfer_between_b200_and_reference_vertices(amb_lib):
    from actionmesh_b200.denoiser import B200Denoiser, DenoiserConfig
    from actionmesh_b200.guidance import ClassifierFreeGuidance
    from actionmesh_b200.scheduler import B200SchedulerFlow

    g = load_golden("denoiser_tiny_multiseed.pt")
    cfg = DenoiserConfig(inflated_layers=tuple(range(g["config"]["num_layers"])), **g["config"])
    acfg, asd, pts, query = _decode_setup()
    sch = B200SchedulerFlow(num_inference_steps=4, shift=3.0, is_additive=True)
    cf = ClassifierFreeGuidance(guidance_at_inference=[[0, 1], [1, 1]], guidance_scales=[7.5])
    rows = []
    for pair in g["pairs"]:
        sd = synth.make_state_dict(cfg, pair["seed"])
        lat, ctx, fs, mask = synth.make_inputs(1, 3, 31, 64, 9, 128, seed=pair["input_seed"])
        ref_tail, ac_tail = pair["denoise4_out"], pair["denoise4_out_autocast_bf16"]   # frames 1.. (frame 0 is observed)
        ref = torch.cat([lat[0, :1], ref_tail])[None]
        eager = torch.cat([lat[0, :1], ac_tail])[None]
        row = {"seed": pair["seed"], "input_seed": pair["input_seed"]}
        for name, fp32 in (("fp32_stream", True), ("bf16_stream", False)):
            model = B200Denoiser(cfg, residual_fp32=fp32).to("cuda")
            model.load_state_dict(sd)
            ours = sch.denoise(model, cf, lat.clone().cuda(), ctx.cuda(), mask=mask.cuda(), framestep=fs).cpu()
            assert torch.equal(ours[0, 0], lat[0, 0])              # observed frame untouched
            row[name + "_latent_rel_err"] = float((ours[0, 1:] - ref_tail).norm() / ref_tail.norm())
            row[name + "_chamfer"], _ = _chamfer_mean(acfg, asd, pts, query, ours, ref, fs)
        row["autocast_latent_rel_err"] = float((ac_tail - ref_tail).norm() / ref_tail.norm())
        row["autocast_chamfer"], _ = _chamfer_mean(acfg, asd, pts, query, eager, ref, fs)
        rows.append(row)
    n = len(rows)
    mean = {k: sum(r[k] for r in rows) / n for k in rows[0] if k not in ("seed", "input_seed")}
    worst = {k: max(r[k] for r in rows) for k in rows[0] if k not in ("seed", "input_seed")}
    report = {"draws": n, "mean": mean, "max": worst, "rows": rows,
              "note": "Chamfer = mean over 3 frames of actionbench-style CD (n=10000, seed 44) vs the reference's fp32 latents "
                      "decoded identically; autocast = the reference's own modules under torch.autocast(bf16)"}
    os.makedirs(REPORT_DIR, exist_ok=True)
    json.dump(report, open(os.path.join(REPORT_DIR, "chamfer_report.json"), "w"), indent=1)
    print("CHAMFER", json.dumps({"mean": mean, "max": worst}))
    assert n >= 8
    # the shipped configuration (fp32 residual stream) against the reference's own mixed-precision recipe, in the mean
    assert mean["fp32_stream_chamfer"] <= 1.25 * mean["autocast_chamfer"], report["mean"]
    assert mean["fp32_stream_latent_rel_err"] <= 1.25 * mean["autocast_latent_rel_err"], report["mean"]
    # the reference-recipe-equivalent bf16 stream must stay in the same band too (it is the same arithmetic class)
    assert mean["bf16_stream_latent_rel_err"] <= 1.25 * mean["autocast_latent_rel_err"], report["mean"]
