"""Texture modality checks that need no GPU: known answers of the float32 restatement (tests/render_texture_ref.py) for the
wrap modes, the filters, the mip chain and the level of detail; the material fallbacks and texture decoding of
`render.texture_shading`; the visualizer's and the C ABI's argument checks (fake pointers, no launch); and the
`--render_texture` command-line plumbing with the pipeline and renderer stubbed."""
import ctypes as C
import io
import logging

import numpy as np
import pytest
import torch
from PIL import Image

import render_texture_ref as tr
from actionmesh_b200 import inference, ops, render
from actionmesh_b200.gltf import GltfVisual, load_glb, write_glb
from actionmesh_b200.pipeline import ActionMeshB200Pipeline, ActionMeshB200PipelineWithMeshInput, Mesh
from test_inference_cpu import N_FACES, N_VERTS, StubPipeline

f32 = np.float32


# ---- restatement known answers --------------------------------------------------------------------------------------------
def _row(values):
    """A 1-row texture whose red channel holds `values`."""
    img = np.zeros((1, len(values), 3), np.uint8)
    img[0, :, 0] = values
    return img


@pytest.mark.parametrize("mode,nearest,linear", [
    (tr.REPEAT, [3, 3, 0, 0, 0, 3], {0.0: 15.0, 1.0: 15.0}),
    (tr.CLAMP_TO_EDGE, [0, 0, 0, 0, 3, 3], {0.0: 0.0, 1.0: 30.0}),
    (tr.MIRRORED_REPEAT, [3, 0, 0, 0, 3, 0], {0.0: 0.0, 1.0: 30.0}),
])
def test_wrap_modes(mode, nearest, linear):
    w = 4
    img = _row([0, 10, 20, 30])
    us = np.array([-1.25, -0.5 / w, 0.0, 0.5 / w, 1.0, 1.75], f32)
    # floor(u w) = -5, -1, 0, 0, 4, 7
    got = tr.sample_level(img, us, np.full(6, 0.5, f32), False, mode, mode)[:, 0]
    np.testing.assert_array_equal(got, 10 * np.array(nearest, f32))
    for u, want in linear.items():  # u w - 1/2 = -0.5 or 3.5: the half-way blend of texels (-1, 0) or (3, 4)
        assert tr.sample_level(img, np.array([u], f32), np.array([0.5], f32), True, mode, mode)[0, 0] == want


def test_wrap_index_formulas():
    i = np.arange(-9, 10)
    np.testing.assert_array_equal(tr.wrap(i, 4, tr.REPEAT), ((i % 4) + 4) % 4)
    np.testing.assert_array_equal(tr.wrap(i, 4, tr.CLAMP_TO_EDGE), np.clip(i, 0, 3))
    np.testing.assert_array_equal(tr.wrap(np.arange(-8, 8), 4, tr.MIRRORED_REPEAT),
                                  [0, 1, 2, 3, 3, 2, 1, 0] * 2)


def test_filters_at_texel_centres_return_the_texels():
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (8, 16, 3), dtype=np.uint8)
    y, x = np.meshgrid(np.arange(8), np.arange(16), indexing="ij")
    u, v = ((x + 0.5) / 16).astype(f32).ravel(), ((y + 0.5) / 8).astype(f32).ravel()
    for linear in (False, True):
        for mode in tr.WRAPS:
            np.testing.assert_array_equal(tr.sample_level(img, u, v, linear, mode, mode), img.reshape(-1, 3).astype(f32))


def test_one_texel_texture():
    img = np.array([[[7, 99, 250]]], np.uint8)
    assert len(tr.mip_chain(img)) == 1 and ops.texture_level_table(1, 1) == [(0, 1, 1)]
    u = np.array([-3.7, -0.2, 0.0, 0.5, 0.999, 1.0, 42.25], f32)
    for linear in (False, True):
        for mode in tr.WRAPS:
            np.testing.assert_array_equal(tr.sample_level(img, u, u[::-1], linear, mode, mode), np.tile([7, 99, 250], (7, 1)))


def test_mip_chain_of_a_5x3_image_by_hand():
    r = np.array([[0, 4, 8, 12, 16], [20, 24, 28, 32, 36], [40, 44, 48, 52, 56]])
    g = np.array([[1, 0, 0, 0, 9], [0, 1, 0, 0, 9], [9, 9, 9, 9, 9]])   # mean 0.5 rounds up; column 4, row 2 are dropped
    b = np.array([[1, 0, 3, 3, 0], [0, 0, 3, 2, 0], [0, 0, 0, 0, 0]])   # mean 0.25 rounds down, 2.75 up
    levels = tr.mip_chain(np.stack([r, g, b], -1).astype(np.uint8))
    assert [lv.shape for lv in levels] == [(3, 5, 3), (1, 2, 3), (1, 1, 3)]
    # level 1: (0+4+20+24+2)//4 = 12, (8+12+28+32+2)//4 = 20; (1+0+0+1+2)//4 = 1, (0+0+0+0+2)//4 = 0; (1+2)//4 = 0, (11+2)//4 = 3
    np.testing.assert_array_equal(levels[1], [[[12, 1, 0], [20, 0, 3]]])
    # level 2 (a 2 x 1 level: the row index clamps): (12+20+12+20+2)//4 = 16, (1+0+1+0+2)//4 = 1, (0+3+0+3+2)//4 = 2
    np.testing.assert_array_equal(levels[2], [[[16, 1, 2]]])
    assert ops.texture_level_table(5, 3) == [(0, 5, 3), (45, 2, 1), (51, 1, 1)]
    assert [(w, h) for _, w, h in ops.texture_level_table(1024, 768)] == [
        (1024 >> k, max(1, 768 >> k)) for k in range(11)]


@pytest.mark.parametrize("L", [0, 1, 2, 5])
def test_level_of_detail_at_the_threshold_and_one_ulp_above(L):
    a_s = f32(3.3)
    at = np.ldexp(a_s, 2 * L).astype(f32)
    above = np.nextafter(at, f32(np.inf))
    lvl, flt = tr.level_of_detail(np.array([at, above]), np.array([a_s, a_s]), np.array([True, True]), 8, tr.NEAREST,
                                  tr.LINEAR_MIPMAP_NEAREST)
    assert lvl.tolist() == [L, L + 1]
    assert flt.tolist() == [tr.NEAREST if L == 0 else tr.LINEAR_MIPMAP_NEAREST, tr.LINEAR_MIPMAP_NEAREST]


def test_level_of_detail_clamps_and_non_mip_modes():
    a_t, a_s = np.array([1e30, 8.0, 8.0], f32), np.array([1.0, 1.0, 1.0], f32)
    pos = np.array([True, True, False])
    lvl, flt = tr.level_of_detail(a_t, a_s, pos, 4, tr.LINEAR, tr.NEAREST_MIPMAP_LINEAR)
    assert lvl.tolist() == [3, 2, 0] and flt.tolist() == [tr.NEAREST_MIPMAP_LINEAR] * 2 + [tr.LINEAR]
    for mn in (tr.NEAREST, tr.LINEAR):
        lvl, flt = tr.level_of_detail(a_t, a_s, pos, 4, tr.LINEAR, mn)
        assert lvl.tolist() == [0, 0, 0] and flt.tolist() == [mn, mn, tr.LINEAR]


# ---- materials and decoding -----------------------------------------------------------------------------------------------
def _png(img: Image.Image) -> bytes:
    buf = io.BytesIO()
    img.save(buf, format="PNG")
    return buf.getvalue()


def _visual(info=None, factor=None, sampler=None, data=None, uv=True):
    pbr = {}
    if factor is not None:
        pbr["baseColorFactor"] = factor
    if info is not None:
        pbr["baseColorTexture"] = info
    tex = {"source": 0}
    if sampler is not None:
        tex["sampler"] = 0
    data = data or _png(Image.new("RGB", (3, 2), (10, 20, 30)))
    return GltfVisual(uv=np.zeros((4, 2), f32) if uv else None, material={"pbrMetallicRoughness": pbr}, textures=[tex],
                      samplers=[sampler] if sampler is not None else [], images=[{"mimeType": "image/png"}],
                      image_bytes=[data])


def test_material_fallbacks(caplog):
    none = render.texture_shading(None)
    assert none.image is None and none.base_color == (0.2, 0.4, 0.8)
    assert render.texture_shading(GltfVisual(uv=np.zeros((4, 2), f32))).base_color == (0.2, 0.4, 0.8)  # no material
    flat = render.texture_shading(_visual(factor=[0.5, 0.25, 1.0, 0.3]))
    assert flat.image is None and flat.base_color == (0.5, 0.25, 1.0)
    assert render.texture_shading(_visual()).base_color == (1.0, 1.0, 1.0)  # glTF's default factor
    tex = render.texture_shading(_visual({"index": 0}, factor=[0.5, 0.5, 0.5, 1.0]))
    assert tex.image.shape == (2, 3, 3) and (tex.image == [10, 20, 30]).all() and tex.base_color == (0.5, 0.5, 0.5)
    assert (tex.mag_filter, tex.min_filter, tex.wrap_s, tex.wrap_t) == (9729, 9985, 10497, 10497)
    assert render.texture_shading(_visual({"index": 0, "texCoord": 0})).image is not None
    smp = render.texture_shading(_visual({"index": 0}, sampler={"magFilter": 9728, "wrapT": 33648}))
    assert (smp.mag_filter, smp.min_filter, smp.wrap_s, smp.wrap_t) == (9728, 9985, 10497, 33648)
    caplog.clear()
    for info, uv, why in (({"index": 0, "texCoord": 1}, True, "texCoord 1"),
                          ({"index": 0, "extensions": {"KHR_texture_transform": {"scale": [2, 2]}}}, True,
                           "KHR_texture_transform"),
                          ({"index": 0}, False, "no UVs")):
        with caplog.at_level(logging.WARNING, logger="actionmesh_b200.render"):
            got = render.texture_shading(_visual(info, factor=[0.1, 0.2, 0.3, 1.0], uv=uv))
        assert got.image is None and got.base_color == (0.1, 0.2, 0.3)
        warnings = [r for r in caplog.records if r.levelno == logging.WARNING]
        assert len(warnings) == 1 and why in warnings[0].getMessage()
        caplog.clear()


def test_bad_samplers_and_sizes_are_refused():
    for smp in ({"magFilter": 9984}, {"minFilter": 1}, {"wrapS": 10496}, {"wrapT": 0}):
        with pytest.raises(ValueError, match="sampler"):
            render.texture_shading(_visual({"index": 0}, sampler=smp))
    with pytest.raises(ValueError, match="16384"):
        render.texture_shading(_visual({"index": 0}, data=_png(Image.new("L", (16385, 1)))))
    assert render.texture_shading(_visual({"index": 0}, data=_png(Image.new("L", (16384, 1))))).image.shape == (1, 16384, 3)
    with pytest.raises(ValueError, match="GltfVisual"):
        render.texture_shading(object())


def test_panda_fixture_texture(golden_dir):
    mesh = load_glb(f"{golden_dir}/panda_blender_small.glb")
    tex = render.texture_shading(mesh.visual)
    assert tex.image.shape == (64, 64, 3) and tex.image.dtype == np.uint8
    assert (tex.mag_filter, tex.min_filter, tex.wrap_s, tex.wrap_t) == (9729, 9987, 10497, 10497)
    assert tex.base_color == (1.0, 1.0, 1.0)
    want = np.array(Image.open(io.BytesIO(mesh.visual.image_bytes[0])).convert("RGB"))
    np.testing.assert_array_equal(tex.image, want)
    assert tex.image.std() > 10  # a real picture


@pytest.mark.parametrize("mode", ["RGBA", "L", "P"])
def test_png_textures_through_a_glb(tmp_path, mode):
    rng = np.random.default_rng(1)
    if mode == "P":
        img = Image.fromarray(rng.integers(0, 16, (5, 7), dtype=np.uint8), "P")
        img.putpalette(rng.integers(0, 256, 48, dtype=np.uint8).tolist())
    else:
        img = Image.fromarray(rng.integers(0, 256, (5, 7, 4) if mode == "RGBA" else (5, 7), dtype=np.uint8), mode)
    vis = GltfVisual(uv=rng.random((3, 2)).astype(f32),
                     material={"pbrMetallicRoughness": {"baseColorTexture": {"index": 0}}},
                     textures=[{"source": 0, "sampler": 0}], samplers=[{"minFilter": 9728, "wrapS": 33071}],
                     images=[{"mimeType": "image/png"}], image_bytes=[_png(img)])
    write_glb(tmp_path / "m.glb", Mesh(vertices=np.eye(3), faces=np.array([[0, 1, 2]]), visual=vis))
    tex = render.texture_shading(load_glb(tmp_path / "m.glb").visual)
    np.testing.assert_array_equal(tex.image, np.array(img.convert("RGB")))
    assert (tex.min_filter, tex.wrap_s) == (9728, 33071)
    if mode == "RGBA":
        np.testing.assert_array_equal(tex.image, np.asarray(img)[..., :3])  # alpha is ignored, not composited


# ---- argument validation --------------------------------------------------------------------------------------------------
class _M:
    def __init__(self, v, f):
        self.vertices, self.faces = v, f


def test_visualizer_validation():
    from actionmesh_b200 import AmbError

    mesh = _M(np.eye(3), [[0, 1, 2]])
    vis = render.B200MeshVisualizer(image_size=8, device="cpu")
    for bad in (("normal", "shaded"), ("texture", "texture"), (), "flat"):
        with pytest.raises(ValueError, match="modalities"):  # before any device work, so before the CPU refusal
            vis.render_frames([mesh], modalities=bad)
        with pytest.raises(ValueError, match="modalities"):
            vis.render([], device="cpu", modalities=bad)
    with pytest.raises(ValueError, match="vertices"):
        vis.render_frames([mesh], modalities=("texture",), visual=GltfVisual(uv=np.zeros((4, 2), f32)))
    with pytest.raises(ValueError, match="non-finite"):
        vis.render_frames([mesh], visual=GltfVisual(uv=np.array([[0, 0], [np.inf, 0], [1, 1]], f32)))
    with pytest.raises(AmbError):
        vis.render_frames([mesh], modalities=("normal", "texture"), visual=GltfVisual(uv=np.zeros((3, 2), f32)))
    assert render.B200MeshVisualizer(image_size=8).render([], modalities=("texture",)) == []


def test_ops_refuse_cpu_tensors():
    from actionmesh_b200 import AmbError

    v, f = torch.eye(3), torch.tensor([[0, 1, 2]], dtype=torch.int32)
    with pytest.raises(AmbError):
        ops.texture_levels(torch.zeros(4, 4, 3, dtype=torch.uint8))
    with pytest.raises(AmbError):
        ops.shade_texture(v, f, v, torch.zeros(1, 12), 2.0, torch.zeros(1, 16, 16, dtype=torch.int32))


def _table(rows):
    flat = [x for r in rows for x in r]
    return (C.c_int64 * max(1, len(flat)))(*flat)


def test_texture_abi_argument_validation(amb_lib):
    """Both texture entry points validate their arguments before any launch (fake non-null pointers)."""
    P = 16
    err = lambda: amb_lib.amb_last_error().decode()  # noqa: E731
    good = ops.texture_level_table(5, 3)
    lv = lambda rows, n=None, buf=P: amb_lib.amb_render_texture_levels(buf, _table(rows), len(rows) if n is None else n,  # noqa: E731
                                                                         None)
    assert lv(good, buf=None) < 0 and "null pointer" in err()
    assert amb_lib.amb_render_texture_levels(P, None, 3, None) < 0 and "null pointer" in err()
    assert lv(good, n=0) < 0 and "n_levels" in err()
    assert lv(ops.texture_level_table(1, 1) * 16, n=16) < 0 and "n_levels" in err()
    assert lv([(0, 16385, 1)] + ops.texture_level_table(8192, 1)) < 0 and "16384" in err()
    assert lv([(0, 0, 3)]) < 0 and "16384" in err()
    assert lv([(0, 5, 3), (45, 3, 1), (54, 1, 1)]) < 0 and "halved" in err()
    assert lv([(0, 5, 3), (40, 2, 1), (51, 1, 1)]) < 0 and "overlap" in err()
    assert lv(good[:2]) < 0 and "1 x 1" in err()
    sh = lambda **k: amb_lib.amb_render_shade_texture(  # noqa: E731
        P, 3, P, 1, P, k.get("uv", P), P, 3, 2.0, 8, P, k.get("lv", P), k.get("tab", _table(good)), k.get("n", 3),
        k.get("mag", 9729), k.get("min", 9985), k.get("ws", 10497), k.get("wt", 10497), 1.0, 1.0, 1.0, k.get("out", P),
        k.get("row", 72), k.get("view", 24), None)
    assert sh(out=None) < 0 and "null pointer" in err()
    assert sh(uv=None) < 0 and "null pointer" in err()
    assert sh(lv=None) < 0 and "null pointer" in err()
    assert sh(tab=None) < 0 and "null pointer" in err()
    assert sh(row=23) < 0 and "bad strides" in err()
    assert sh(view=23) < 0 and "bad strides" in err()
    for name, bad in (("mag", 9987), ("min", 9983), ("min", 9988), ("ws", 33072), ("wt", 0)):
        assert sh(**{name: bad}) < 0 and "bad " in err() and str(bad) in err()
    assert sh(n=2) < 0 and "1 x 1" in err()
    assert sh(n=-1) < 0 and "n_levels" in err()
    assert sh(n=0, uv=None, lv=None, tab=None, mag=1) < 0 and "mag_filter" in err()  # enums are checked without a texture


# ---- the command line -----------------------------------------------------------------------------------------------------
@pytest.fixture
def stubs(monkeypatch):
    built, rendered = [], []

    def factory(cls):
        def from_pretrained(*args, **kwargs):
            built.append(StubPipeline(cls, args, kwargs))
            return built[-1]
        return from_pretrained

    class Visualizer:
        def __init__(self, image_size=256):
            self.image_size = image_size

        def render(self, meshes, device, output_dir, input_frames, **kwargs):
            rendered.append(dict(meshes=meshes, device=device, output_dir=output_dir, **kwargs))

    for cls in (ActionMeshB200Pipeline, ActionMeshB200PipelineWithMeshInput):
        monkeypatch.setattr(cls, "from_pretrained", classmethod(lambda c, *a, **k: factory(c)(*a, **k)))
    monkeypatch.setattr(render, "B200MeshVisualizer", Visualizer)
    return built, rendered


@pytest.fixture
def frames_dir(tmp_path):
    d = tmp_path / "clip"
    d.mkdir()
    for i in range(16):  # the pipeline's minimum clip
        Image.fromarray(np.random.default_rng(i).integers(0, 255, (32, 32, 4), dtype=np.uint8), "RGBA").save(d / f"{i}.png")
    return d


def test_render_texture_flag(stubs, frames_dir, tmp_path):
    _, rendered = stubs
    inference.main(["--input", str(frames_dir), "--output_dir", str(tmp_path / "a")])
    inference.main(["--input", str(frames_dir), "--output_dir", str(tmp_path / "b"), "--render_texture"])
    plain, textured = rendered
    assert set(plain) == {"meshes", "device", "output_dir"}  # without the flag: the normal-only call, unchanged
    assert textured["modalities"] == ("normal", "texture") and textured["visual"] is None


def test_render_texture_flag_with_mesh_input(stubs, frames_dir, tmp_path):
    built, rendered = stubs
    rng = np.random.default_rng(5)
    visual = GltfVisual(uv=rng.random((N_VERTS, 2)).astype(f32),
                        material={"pbrMetallicRoughness": {"baseColorTexture": {"index": 0}}},
                        textures=[{"source": 0}], images=[{"mimeType": "image/png"}],
                        image_bytes=[_png(Image.new("RGB", (4, 4), (1, 2, 3)))])
    write_glb(tmp_path / "in.glb", Mesh(vertices=rng.standard_normal((N_VERTS, 3)),
                                        faces=rng.integers(0, N_VERTS, (N_FACES, 3)), visual=visual))
    inference.main(["--input", str(frames_dir), "--mesh_input", str(tmp_path / "in.glb"), "--output_dir",
                    str(tmp_path / "out"), "--render_texture"])
    (r,) = rendered
    assert built[0].calls[0]["anchor_mesh"].visual is None      # the pipeline dropped it in place ...
    assert r["modalities"] == ("normal", "texture")             # ... but the render gets the input's
    np.testing.assert_array_equal(r["visual"].uv, visual.uv)
    assert r["visual"].material == visual.material and r["visual"].image_bytes == visual.image_bytes
    assert all(len(m.vertices) == N_VERTS for m in r["meshes"])
