"""The mesh-input encoder path without a GPU: the fp32 encoder restatement and the numpy farthest-point sampling against the
reference's own TripoSG VAE encoder (golden), and the encoder-side state-dict keys."""
import numpy as np
import torch

import triposg_vae_encoder_ref as ref
from conftest import load_golden


def _golden():
    g = load_golden("triposg_vae_encoder_tiny.pt")
    c = g["config"]
    sd = ref.make_encoder_state_dict(c["width_encoder"], c["num_attention_heads"], c["num_layers_encoder"], seed=g["seed"])
    return g, c, sd


def test_subset_is_the_reference_rng_choice():
    g, _, _ = _golden()
    n, m = g["surface"].shape[1], 4 * g["num_tokens"]
    subset = np.random.default_rng(g["subset_seed"]).choice(n, m, replace=m > n)
    assert np.array_equal(subset, g["subset"].numpy())


def test_numpy_fps_matches_golden_indices():
    g, _, _ = _golden()
    xyz = g["surface"][0, g["subset"], :3].numpy()
    idx = ref.fps_numpy(xyz, g["num_tokens"], g["fps_start"])
    assert np.array_equal(idx, g["fps_index"].numpy())
    assert idx[0] == g["fps_start"] and len(np.unique(idx)) == len(idx)


def test_numpy_fps_ties_and_exhaustion():
    pts = np.zeros((6, 3), dtype=np.float32)
    pts[3] = 1.0
    pts[4] = 0.5
    pts[5] = 1.0                      # duplicate of point 3: the lower index wins the tie
    assert ref.fps_numpy(pts, 5, 0).tolist() == [0, 3, 4, 0, 0]   # then every distance is 0: argmax repeats index 0


def test_fp32_encoder_restatement_matches_reference():
    g, c, sd = _golden()
    surface = g["surface"]
    sampled = surface[:, g["subset"]][:, g["fps_index"]]
    quant = ref.encode_fp32(sd, surface, sampled, c["num_attention_heads"], c["num_layers_encoder"])
    err = float((quant - g["quant"]).norm() / g["quant"].norm())
    assert quant.shape == g["quant"].shape == (1, 256, 128) and err <= 1e-5, err
    lat = ref.posterior_sample(quant, g["eps"])
    err = float((lat - g["latent"]).norm() / g["latent"].norm())
    assert err <= 1e-5, err


def test_encoder_state_dict_keys():
    keys = set(ref.make_encoder_state_dict(256, 4, 2))
    assert {k.split(".")[0] for k in keys} == {"encoder", "quant"}
    assert "encoder.blocks.0.attn2.norm_cross.weight" in keys and "encoder.blocks.2.attn1.to_q.weight" in keys
    assert "encoder.blocks.0.attn1.to_q.weight" not in keys and "encoder.blocks.3.norm1.weight" not in keys


def test_encoder_config_checks():
    from actionmesh_b200.triposg_vae import TripoSGVAEConfig

    assert TripoSGVAEConfig().encoder_supported() is None                      # 512 wide, 8 heads x 64
    assert TripoSGVAEConfig().encoder_in_dim == 54
    assert TripoSGVAEConfig(width_decoder=256, num_attention_heads=2).encoder_supported() is not None   # 512 / 2 = 256
    assert TripoSGVAEConfig(width_encoder=256, width_decoder=512, num_attention_heads=4).encoder_supported() is None
