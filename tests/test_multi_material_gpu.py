"""Per-face material shading against the float32 restatement (tests/render_materials_ref.py), bit for bit (-m gpu): seeded
triangle soups with 1, 7 and 300 records over every wrap x filter pair, three chains packed in one buffer and flat
records, at S in {8, 50, 256}; the panda split into four primitives over 8 frames; one record against `shade_texture`;
a multi-material mesh input through the command line's whole path."""
import numpy as np
import pytest
import torch

import glb_check
import render_materials_ref as mr
import render_texture_ref as tr
from render_ref import vertex_normals_ref
from test_multi_material_cpu import png, split
from test_render_gpu import _cams, _soup
from test_render_texture_gpu import _golden, _texture, _uv

pytestmark = pytest.mark.gpu

WRAP_PAIRS = [(s, t) for s in tr.WRAPS for t in tr.WRAPS]
CHAINS = [(1, 1), (53, 37), (768, 1024)]  # (h, w)


def _packed_chains(images):
    """Every image's chain in one level buffer -> (levels, tables)."""
    from actionmesh_b200 import ops

    sizes = [ops.texture_chain_bytes(im.shape[1], im.shape[0]) for im in images]
    levels = torch.empty(sum(sizes), dtype=torch.uint8, device="cuda")
    tables, off = [], 0
    for im, size in zip(images, sizes):
        tables.append(ops.texture_levels(torch.from_numpy(im).cuda(), out=levels, offset=off)[1])
        off += size
    return levels, tables


@pytest.mark.parametrize("S", [8, 50, 256])
@pytest.mark.parametrize("n_records", [1, 7, 300])
def test_soup_bit_exact(amb_lib, S, n_records):
    """Record k: chain k % 4 (the fourth is flat), wrap pair k % 9, minFilter (k // 9) % 6, magFilter (k // 54) % 2 -- with
    300 records every wrap x filter pair appears."""
    from actionmesh_b200 import ops

    case = [8, 50, 256].index(S) * 3 + [1, 7, 300].index(n_records)
    cams, focal = _cams()
    v, f = _soup(case, n=320 if n_records == 300 else (48 if S < 256 else 24))
    uv = _uv(case, len(v) // 3)
    rng = np.random.default_rng(case)
    images = [_texture(h, w, seed=case + k) for k, (h, w) in enumerate(CHAINS)]
    levels, tables = _packed_chains(images)
    chains = [tr.mip_chain(im) for im in images]
    rows, ref_records = [], []
    for k in range(n_records):
        c = (k + case) % 4
        sampler = ((tr.NEAREST, tr.LINEAR)[(k // 54 + case) % 2], tr.MIN_FILTERS[(k // 9) % 6]) + WRAP_PAIRS[k % 9]
        base = tuple(float(x) for x in rng.uniform(0.2, 1.0, 3))
        rows.append((tables[c] if c < 3 else None, *sampler, base))
        ref_records.append((chains[c] if c < 3 else None, sampler, base))
    face_record = rng.integers(0, n_records, len(f))
    vt, ft, ct = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(cams).cuda()
    normals = ops.vertex_normals(vt, ft)
    p2f = ops.rasterize(vt, ft, ct, focal, S)
    got = ops.shade_materials(vt, ft, normals, ct, focal, p2f, ops.face_records(face_record, n_records, "cuda"),
                              ops.shade_records(rows, levels, "cuda"), levels, torch.from_numpy(uv).cuda())
    got = got.cpu().numpy().reshape(S, len(cams), S, 3).transpose(1, 0, 2, 3)
    p2f_h = p2f.cpu().numpy()
    want = mr.shade_materials_ref(v, f, vertex_normals_ref(v, f), uv, cams, focal, S, p2f_h, face_record, ref_records)
    np.testing.assert_array_equal(got, want)
    hit = np.unique(face_record[p2f_h[p2f_h >= 0]])
    assert (p2f_h >= 0).mean() > 0.5 and len(hit) >= min(n_records, 100)


def _panda_split(n_frames):
    """The panda fixture as four primitives: its own texture, a second texture with CLAMP_TO_EDGE and NEAREST, a
    factor-only material and a material-less, UV-less primitive; deformed over `n_frames` as test_render_texture_gpu's
    panda -> (meshes, visual)."""
    from actionmesh_b200.gltf import GltfMultiVisual, load_glb
    from test_render_texture_gpu import _M

    mesh = load_glb(_golden("panda_blender_small.glb"))
    pv = mesh.visual
    F = len(mesh.faces)
    groups = np.array_split(np.random.default_rng(0).permutation(F), 4)
    verts, faces, uv, vr, fr = split(mesh.vertices, mesh.faces, pv.uv, [np.sort(g) for g in groups])
    uv[vr[3, 0]:] = 0
    second = png(np.random.default_rng(9).integers(0, 256, (48, 64, 3), dtype=np.uint8))
    materials = [pv.material, {"pbrMetallicRoughness": {"baseColorTexture": {"index": len(pv.textures)},
                                                        "baseColorFactor": [0.9, 0.8, 1.0, 1.0]}},
                 {"pbrMetallicRoughness": {"baseColorFactor": [0.3, 0.7, 0.2, 1.0]}}]
    visual = GltfMultiVisual(vertex_ranges=vr, face_ranges=fr, uv=uv, has_uv=np.array([True, True, True, False]),
                             primitive_material=[0, 1, 2, None], materials=materials,
                             textures=pv.textures + [{"sampler": len(pv.samplers), "source": len(pv.images)}],
                             samplers=pv.samplers + [{"magFilter": 9728, "minFilter": 9728, "wrapS": 33071, "wrapT": 33071}],
                             images=pv.images + [{"mimeType": "image/png"}], image_bytes=pv.image_bytes + [second])
    base = verts - np.array([0.09, 0.05, 0.0])
    out = []
    for k in range(n_frames):
        a = 0.08 * k * base[:, 1]
        x, z = base[:, 0] * np.cos(a) - base[:, 2] * np.sin(a), base[:, 0] * np.sin(a) + base[:, 2] * np.cos(a)
        out.append(_M(np.stack([x, base[:, 1] + 0.02 * k, z], 1), faces))
    return out, visual


def _materials_ref_grid(meshes, visual, S):
    """The restatement's cells of every mesh, with pix_to_face from the (separately checked) GPU rasterizer."""
    from actionmesh_b200 import ops
    from actionmesh_b200.render import _mesh_arrays, texture_shading

    cams, focal = _cams()
    sh = texture_shading(visual)
    chains = [tr.mip_chain(im) for im in sh.images]
    records = [(None if r.image is None else chains[r.image], (r.mag_filter, r.min_filter, r.wrap_s, r.wrap_t),
                r.base_color) for r in sh.records]
    out = []
    for m in meshes:
        v, f, keep = _mesh_arrays(m)
        f = f[keep].astype(np.int32)
        p2f = ops.rasterize(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(cams).cuda(), focal,
                            S).cpu().numpy()
        cells = mr.shade_materials_ref(v, f, vertex_normals_ref(v, f), visual.uv, cams, focal, S, p2f,
                                       sh.face_record[keep], records)
        out.append(np.concatenate(list(cells), axis=1))
    return np.stack(out)


def test_panda_split_over_8_frames_whole_grid(amb_lib):
    from actionmesh_b200.render import B200MeshVisualizer

    S = 256
    meshes, visual = _panda_split(8)
    vis = B200MeshVisualizer(image_size=S)
    grid = vis.render_frames(meshes, modalities=("texture",), visual=visual).numpy()
    assert grid.shape == (8, S, 3 * S, 3)
    np.testing.assert_array_equal(grid, _materials_ref_grid(meshes, visual, S))
    assert (grid != 255).any(axis=-1).mean() > 0.02
    again = vis.render_frames(meshes, modalities=("texture",), visual=visual).numpy()
    assert again.tobytes() == grid.tobytes()


def test_one_record_equals_shade_texture(amb_lib):
    """One record over every face shades exactly as `shade_texture` with that record: the panda's texture, and flat."""
    from actionmesh_b200 import ops
    from actionmesh_b200.gltf import load_glb
    from actionmesh_b200.render import mesh_arrays, texture_shading

    mesh = load_glb(_golden("panda_blender_small.glb"))
    sh = texture_shading(mesh.visual)
    cams, focal = _cams()
    v, f = mesh_arrays(mesh)
    vt, ft, ct = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(cams).cuda()
    normals = ops.vertex_normals(vt, ft)
    p2f = ops.rasterize(vt, ft, ct, focal, 256)
    levels, table = ops.texture_levels(torch.from_numpy(sh.image).cuda())
    uv = torch.from_numpy(mesh.visual.uv).cuda()
    mode = dict(mag_filter=sh.mag_filter, min_filter=sh.min_filter, wrap_s=sh.wrap_s, wrap_t=sh.wrap_t)
    face_record = ops.face_records(np.zeros(len(f), np.int32), 1, "cuda")
    for tex in (True, False):
        want = ops.shade_texture(vt, ft, normals, ct, focal, p2f, *((uv, levels, table) if tex else ()),
                                 base_color=sh.base_color, **mode)
        rec = ops.shade_records([(table if tex else None, *mode.values(), sh.base_color)], levels, "cuda")
        n0 = ops.launch_count
        got = ops.shade_materials(vt, ft, normals, ct, focal, p2f, face_record, rec, levels, uv)
        assert ops.launch_count - n0 == 1
        assert got.cpu().numpy().tobytes() == want.cpu().numpy().tobytes()
        assert (want.cpu().numpy() != 255).any()


def test_multi_material_mesh_input_end_to_end(tmp_path, amb_lib):
    """A multi-material --mesh_input through the command line's path on the tiny checkpoint tree: both GLBs carry the
    input's materials, and mesh_XX.glb, the deformation arrays and the normal video are those of the same file with its
    materials and UVs stripped."""
    import standalone_tree as st
    from actionmesh_b200.gltf import GltfMultiVisual, load_glb, write_glb
    from actionmesh_b200.inference import run_actionmesh
    from actionmesh_b200.pipeline import ActionMeshB200PipelineWithMeshInput, Mesh
    from test_inference_gpu import UPDATES, _frames_dir, _video_frames

    root = st.centred_tree(str(tmp_path / "pretrained_weights"))
    sphere = st.textured_sphere()
    F = len(sphere.faces)
    verts, faces, uv, vr, fr = split(sphere.vertices, sphere.faces, sphere.visual.uv, [np.arange(F // 2), np.arange(F // 2, F)])
    sv = sphere.visual
    visual = GltfMultiVisual(vertex_ranges=vr, face_ranges=fr, uv=uv, has_uv=np.array([True, False]),
                             primitive_material=[0, 1], materials=[sv.material, {"pbrMetallicRoughness": {
                                 "baseColorFactor": [0.8, 0.1, 0.1, 1.0]}}],
                             textures=sv.textures, samplers=sv.samplers, images=sv.images, image_bytes=sv.image_bytes)
    visual.uv[vr[1, 0]:] = 0
    write_glb(tmp_path / "multi.glb", Mesh(verts, faces, visual))
    write_glb(tmp_path / "plain.glb", Mesh(verts, faces))
    assert isinstance(load_glb(tmp_path / "multi.glb").visual, GltfMultiVisual)
    frames = _frames_dir(tmp_path, 16)
    updates = {**UPDATES, "model.temporal_3D_denoiser.num_tokens_nominal": 2048}
    pipe = ActionMeshB200PipelineWithMeshInput.from_pretrained(root, config_updates=updates).to("cuda")
    outs = {}
    for name in ("multi", "plain"):
        outs[name] = tmp_path / f"out_{name}"
        run_actionmesh(pipe, str(frames), str(outs[name]), seed=44, mesh_input=str(tmp_path / f"{name}.glb"),
                       render_texture=True, skinning_bones=4)
    want = load_glb(tmp_path / "multi.glb").visual
    for glb in ("animated_mesh.glb", "skinned_mesh.glb"):
        gltf, binary = glb_check.check_glb(outs["multi"] / glb) if glb == "animated_mesh.glb" else _check_skinned(outs["multi"] / glb)
        prims = gltf["meshes"][0]["primitives"]
        assert len(prims) == 2 and gltf["materials"][prims[0]["material"]] == want.materials[0]
        assert gltf["materials"][prims[1]["material"]] == want.materials[1]
        assert "TEXCOORD_0" in prims[0]["attributes"] and "TEXCOORD_0" not in prims[1]["attributes"]
        assert glb_check.image_bytes(gltf, binary) == want.image_bytes
    names = sorted(p.name for p in outs["plain"].iterdir() if p.name.startswith("mesh_") or p.suffix == ".npy")
    assert len(names) == 16 + 2
    for name in names:
        assert (outs["multi"] / name).read_bytes() == (outs["plain"] / name).read_bytes(), name
    assert np.array_equal(_video_frames(outs["multi"] / "grid_normal.mp4"), _video_frames(outs["plain"] / "grid_normal.mp4"))
    tex = [_video_frames(outs[n] / "grid_texture.mp4") for n in ("multi", "plain")]
    assert tex[0].shape == tex[1].shape and not np.array_equal(tex[0], tex[1])


def _check_skinned(path):
    old = glb_check.NCOMP.get("MAT4")
    glb_check.NCOMP["MAT4"] = 16
    try:
        return glb_check.check_glb(path)
    finally:
        if old is None:
            del glb_check.NCOMP["MAT4"]
