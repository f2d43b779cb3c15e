"""The texture modality's kernels against the float32 restatement (tests/render_texture_ref.py), bit for bit (-m gpu): mip
levels; seeded triangle soups with uv in [-2, 3] over every wrapS x wrapT, both magFilters and all six minFilters, on 1 x 1,
37 x 53 and 1024 x 768 textures at S in {8, 50, 256}; the panda fixture deformed over 8 frames; determinism; the normal grid
of a two-modality call; the default colour; launch counts."""
import numpy as np
import pytest
import torch

import render_texture_ref as tr
from render_ref import rasterize_ref, vertex_normals_ref
from test_render_gpu import _cams, _soup

pytestmark = pytest.mark.gpu

WRAP_PAIRS = [(s, t) for s in tr.WRAPS for t in tr.WRAPS]


class _M:
    def __init__(self, v, f):
        self.vertices, self.faces = v, f


def _texture(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("hw", [(1, 1), (3, 5), (53, 37), (768, 1024), (1, 300)])
def test_mip_levels_byte_equal(amb_lib, hw):
    from actionmesh_b200 import ops

    img = _texture(*hw, seed=hw[0])
    levels, table = ops.texture_levels(torch.from_numpy(img).cuda())
    got = levels.cpu().numpy()
    want = tr.mip_chain(img)
    assert len(table) == len(want)
    for (off, w, h), lv in zip(table, want):
        np.testing.assert_array_equal(got[off:off + 3 * w * h].reshape(h, w, 3), lv)


def _uv(seed, n_faces):
    """Per-corner uv in [-2, 3]: each face around its own centre, with spreads from 1e-4 to 2 so that faces are magnified
    and minified by every factor."""
    rng = np.random.default_rng(seed)
    centre = rng.uniform(-2, 3, (n_faces, 1, 2))
    spread = 10 ** rng.uniform(-4, np.log10(2), (n_faces, 1, 1))
    return np.clip(centre + spread * rng.uniform(-1, 1, (n_faces, 3, 2)), -2, 3).astype(np.float32).reshape(-1, 2)


@pytest.mark.parametrize("S", [8, 50, 256])
@pytest.mark.parametrize("tex_hw", [(1, 1), (53, 37), (768, 1024)])
def test_soup_bit_exact(amb_lib, S, tex_hw):
    from actionmesh_b200 import ops

    case = [8, 50, 256].index(S) * 3 + [(1, 1), (53, 37), (768, 1024)].index(tex_hw)
    cams, focal = _cams()
    v, f = _soup(case, n=48 if S < 256 else 24)
    uv = _uv(case, len(v) // 3)  # the soup's faces own their corners
    img = _texture(*tex_hw, seed=case)
    vt, ft, ct = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(cams).cuda()
    normals = ops.vertex_normals(vt, ft)
    p2f = ops.rasterize(vt, ft, ct, focal, S)
    levels, table = ops.texture_levels(torch.from_numpy(img).cuda())
    p2f_h = p2f.cpu().numpy()
    np.testing.assert_array_equal(p2f_h, rasterize_ref(v, f, cams, focal, S))
    nrm = vertex_normals_ref(v, f)
    chain = tr.mip_chain(img)
    uvt = torch.from_numpy(uv).cuda()
    used = set()
    for k, mn in enumerate(tr.MIN_FILTERS):  # every minFilter here; the wrap pairs cycle through all nine over the cases
        mag = (tr.NEAREST, tr.LINEAR)[(k + case) % 2]
        ws, wt = WRAP_PAIRS[(6 * case + k) % 9]
        base = (1.0, 0.75, 0.5) if k % 3 else (1.0, 1.0, 1.0)
        got = ops.shade_texture(vt, ft, normals, ct, focal, p2f, uvt, levels, table, mag_filter=mag, min_filter=mn,
                                wrap_s=ws, wrap_t=wt, base_color=base)
        got = got.cpu().numpy().reshape(S, len(cams), S, 3).transpose(1, 0, 2, 3)
        want = tr.shade_texture_ref(v, f, nrm, uv, cams, focal, S, p2f_h, chain, (mag, mn, ws, wt), base)
        np.testing.assert_array_equal(got, want, err_msg=f"mag {mag} min {mn} wrap {ws} {wt}")
        used.add((ws, wt))
    assert (p2f_h >= 0).mean() > 0.5 and len(used) == 6


def test_several_levels_are_used(amb_lib):
    """On the 1024 x 768 texture at S = 50 the soup's faces reach many mip levels and both filter paths."""
    cams, focal = _cams()
    S = 50
    v, f = _soup(5, n=48)  # test_soup_bit_exact's case for this texture and S
    uv = _uv(5, len(v) // 3)
    p2f = rasterize_ref(v, f, cams, focal, S)
    levels_hit = set()
    from render_ref import edge, project

    for c, cam in enumerate(cams):
        faces = np.unique(p2f[c][p2f[c] >= 0])
        pv = project(v, cam, focal)
        fc = f[faces]
        v0, v1, v2 = (pv[fc[:, k]].T for k in range(3))
        t0, t1, t2 = (uv[fc[:, k]] for k in range(3))
        a_s = (np.float32(0.5) * np.abs(edge(v0[0], v0[1], v1, v2))) * np.float32(S * S)
        a_t = (np.float32(0.5) * np.abs(edge(t0[:, 0], t0[:, 1], t1.T, t2.T))) * np.float32(1024 * 768)
        pos = (v0[2] > 0) & (v1[2] > 0) & (v2[2] > 0)
        lvl, _ = tr.level_of_detail(a_t, a_s, pos, 11, tr.LINEAR, tr.LINEAR_MIPMAP_NEAREST)
        levels_hit |= set(lvl.tolist())
    assert len(levels_hit) >= 4 and 0 in levels_hit


def _panda_frames(n):
    from actionmesh_b200.gltf import load_glb

    mesh = load_glb(_golden("panda_blender_small.glb"))
    base = np.asarray(mesh.vertices) - np.array([0.09, 0.05, 0.0])
    out = []
    for k in range(n):  # a twist about +Y growing with k, and a bob
        a = 0.08 * k * base[:, 1]
        x, z = base[:, 0] * np.cos(a) - base[:, 2] * np.sin(a), base[:, 0] * np.sin(a) + base[:, 2] * np.cos(a)
        out.append(_M(np.stack([x, base[:, 1] + 0.02 * k, z], 1), np.asarray(mesh.faces)))
    return out, mesh.visual


def _golden(name):
    import os

    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name)


def _texture_ref_grid(meshes, visual, S):
    """The restatement's texture cells of every mesh, with pix_to_face from the (separately checked) GPU rasterizer."""
    from actionmesh_b200 import ops
    from actionmesh_b200.render import mesh_arrays, texture_shading

    cams, focal = _cams()
    sh = texture_shading(visual)
    chain = tr.mip_chain(sh.image) if sh.image is not None else None
    uv = None if visual is None else np.asarray(visual.uv, np.float32)
    out = []
    for m in meshes:
        v, f = mesh_arrays(m)
        p2f = ops.rasterize(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(cams).cuda(), focal,
                            S).cpu().numpy()
        cells = tr.shade_texture_ref(v, f, vertex_normals_ref(v, f), uv, cams, focal, S, p2f, chain,
                                     (sh.mag_filter, sh.min_filter, sh.wrap_s, sh.wrap_t), sh.base_color)
        out.append(np.concatenate(list(cells), axis=1))
    return np.stack(out)


def test_panda_over_8_frames_whole_grid(amb_lib):
    from actionmesh_b200.render import B200MeshVisualizer

    S = 256
    meshes, visual = _panda_frames(8)
    vis = B200MeshVisualizer(image_size=S)
    grid = vis.render_frames(meshes, modalities=("texture",), visual=visual).numpy()
    assert grid.shape == (8, S, 3 * S, 3)
    want = _texture_ref_grid(meshes, visual, S)
    np.testing.assert_array_equal(grid, want)
    assert (grid != 255).any(axis=-1).mean() > 0.02  # the panda (a thin half figure) covers about 4 % of the cells
    again = vis.render_frames(meshes, modalities=("texture",), visual=visual).numpy()
    assert again.tobytes() == grid.tobytes()


def test_two_modalities_and_the_files(amb_lib, tmp_path):
    import cv2
    from PIL import Image

    from actionmesh_b200.render import B200MeshVisualizer

    S = 64
    meshes, visual = _panda_frames(5)
    frames = [Image.fromarray(np.full((40, 60, 3), 40 * k, np.uint8)) for k in range(5)]
    vis = B200MeshVisualizer(image_size=S)
    normal, texture = vis.render_frames(meshes, frames, modalities=("normal", "texture"), visual=visual)
    assert normal.numpy().tobytes() == vis.render_frames(meshes, frames).numpy().tobytes()
    tex_only = vis.render_frames(meshes, frames, modalities=("texture",), visual=visual)
    assert texture.numpy().tobytes() == tex_only.numpy().tobytes()
    np.testing.assert_array_equal(texture[:, :, :S], normal[:, :, :S])  # the same input-frame column
    tex_first = vis.render_frames(meshes, modalities=("texture", "normal"), visual=visual)
    np.testing.assert_array_equal(tex_first[0], texture[:, :, S:])
    paths = vis.render(meshes, device="cuda", output_dir=str(tmp_path), input_frames=frames,
                       modalities=("normal", "texture"), visual=visual)
    assert paths == [tmp_path / "grid_normal.mp4", tmp_path / "grid_texture.mp4"]
    for p in paths:
        cap = cv2.VideoCapture(str(p))
        n = 0
        while True:
            ok, fr = cap.read()
            if not ok:
                break
            assert fr.shape == (S, 4 * S, 3)
            n += 1
        cap.release()
        assert n == 5


def test_untextured_mesh_gets_the_default_colour(amb_lib):
    from actionmesh_b200.render import B200MeshVisualizer

    S = 32
    meshes, _ = _panda_frames(2)
    grid = B200MeshVisualizer(image_size=S).render_frames(meshes, modalities=("texture",)).numpy()
    np.testing.assert_array_equal(grid, _texture_ref_grid(meshes, None, S))
    px = grid.reshape(-1, 3).astype(np.float64)
    # red <= 0.2 x 255 only where all four samples hit the mesh (a white sample adds at least 255 / 4); there the colour is
    # (0.2, 0.4, 0.8) times the mean headlight (>= 0.35), truncated
    full = px[(px[:, 0] <= 51) & (px[:, 2] >= 100)]
    assert len(full) > 50
    np.testing.assert_allclose(full / full[:, 2:3], np.broadcast_to([0.25, 0.5, 1.0], full.shape), atol=0.02)


def test_launch_counts(amb_lib):
    from actionmesh_b200 import ops
    from actionmesh_b200.render import B200MeshVisualizer

    meshes, visual = _panda_frames(3)
    vis = B200MeshVisualizer(image_size=16)
    n_levels = len(ops.texture_level_table(64, 64))
    for mods, per_frame, once in ((("normal",), 18, 0), (("texture",), 18, n_levels - 1),
                                  (("normal", "texture"), 19, n_levels - 1)):
        n0 = ops.launch_count
        vis.render_frames(meshes, modalities=mods, visual=visual)
        assert ops.launch_count - n0 == once + 3 * per_frame, mods
    n0 = ops.launch_count
    vis.render_frames(meshes, modalities=("normal", "texture"))  # no texture: no mip chain
    assert ops.launch_count - n0 == 3 * 19


def test_cpu_inputs_are_refused(amb_lib):
    from actionmesh_b200 import AmbError, ops

    cams, focal = _cams()
    v, f = _soup(0, n=8)
    vt, ft, ct = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(cams).cuda()
    p2f = ops.rasterize(vt, ft, ct, focal, 8)
    levels, table = ops.texture_levels(torch.from_numpy(_texture(4, 4, 0)).cuda())
    uv = torch.zeros(len(v), 2, device="cuda")
    with pytest.raises(AmbError):
        ops.shade_texture(vt, ft, ops.vertex_normals(vt, ft), ct, focal, p2f, uv.cpu(), levels, table)
    with pytest.raises(AmbError):
        ops.shade_texture(vt, ft, ops.vertex_normals(vt, ft), ct, focal, p2f, uv, levels.cpu(), table)
