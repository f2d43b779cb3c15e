"""The normal renderer's kernels against the float32 restatement (tests/render_ref.py), bit for bit (-m gpu): seeded
triangle soups with slivers, box-straddling, screen-filling, camera-crossing, coplanar and degenerate faces at S in
{8, 50, 100, 256}; vertex normals; a depth-9 Stage 0 mesh over 16 frames at sampled pixels; determinism; the visualizer's
video; CPU refusal; launch counts."""
import numpy as np
import pytest
import torch

from render_ref import camera_table, rasterize_pairs_ref, render_ref, shade_ref, vertex_normals_ref

pytestmark = pytest.mark.gpu


def _cams():
    from actionmesh_b200.render import uniform_cameras

    c = uniform_cameras()
    return camera_table({t: c[t] for t in ("U000", "U004", "U008")})


def _soup(seed: int, n: int = 48):
    """Random faces in the unit box plus adversarial ones; every face has three distinct corners."""
    rng = np.random.default_rng(seed)
    tris = [rng.uniform(-0.9, 0.9, (3,)) + rng.normal(0, 0.25, (3, 3)) for _ in range(n)]
    for _ in range(6):  # slivers: a third corner within 1e-4 of an edge
        a, b = rng.uniform(-0.8, 0.8, (2, 3))
        tris.append(np.stack([a, b, (a + b) / 2 + rng.normal(0, 1e-4, 3)]))
    for _ in range(4):  # sub-sample faces
        a = rng.uniform(-0.7, 0.7, 3)
        tris.append(a + rng.normal(0, 2e-3, (3, 3)))
    tris.append(np.array([[-40.0, -40.0, -1.2], [40.0, -40.0, -1.2], [0.0, 40.0, -1.2]]))  # fills every screen, far side
    tris.append(np.array([[-30.0, 0.2, -30.0], [30.0, 0.2, -30.0], [0.0, 0.2, 30.0]]))    # plane through the scene
    tris.append(np.array([[0.0, 0.0, 0.0], [5.0, 5.0, 5.0], [-5.0, 5.0, 5.0]]))           # crosses the cameras' planes
    tris.append(tris[3].copy())                                                            # coplanar duplicate: tie
    tris.append(np.array([[0.1, 0.1, 0.1], [0.2, 0.2, 0.2], [0.3, 0.3, 0.3]]))            # collinear: zero area
    v = np.concatenate(tris).astype(np.float32)
    f = np.arange(len(v), dtype=np.int32).reshape(-1, 3)
    return v, f[rng.permutation(len(f))]


def _mesh(seed: int, n_vertices: int = 300, n_faces: int = 900):
    """Random indexed mesh with shared vertices (distinct corners per face)."""
    rng = np.random.default_rng(seed)
    v = rng.uniform(-0.8, 0.8, (n_vertices, 3)).astype(np.float32)
    f = np.stack([rng.choice(n_vertices, 3, replace=False) for _ in range(n_faces)]).astype(np.int32)
    return v, f


def _gpu_render(v, f, cams, focal, S):
    from actionmesh_b200 import ops

    vt, ft, ct = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(cams).cuda()
    normals = ops.vertex_normals(vt, ft)
    p2f = ops.rasterize(vt, ft, ct, focal, S)
    rgb = ops.shade_normals(vt, ft, normals, ct, focal, p2f)
    torch.cuda.synchronize()
    C = len(cams)
    return normals.cpu().numpy(), p2f.cpu().numpy(), rgb.cpu().numpy().reshape(S, C, S, 3).transpose(1, 0, 2, 3)


@pytest.mark.parametrize("S", [8, 50, 100, 256])
@pytest.mark.parametrize("seed", [0, 1])
def test_soup_bit_exact(amb_lib, S, seed):
    cams, focal = _cams()
    v, f = _soup(seed, n=48 if S < 256 else 24)
    normals, p2f, rgb = _gpu_render(v, f, cams, focal, S)
    want_p2f, want_mask, want_rgb = render_ref(v, f, cams, focal, S)
    np.testing.assert_array_equal(p2f, want_p2f)
    np.testing.assert_array_equal(normals.view(np.int32), vertex_normals_ref(v, f).view(np.int32))
    np.testing.assert_array_equal(rgb, want_rgb)
    cov = (p2f >= 0).reshape(len(cams), S, 2, S, 2).sum(axis=(2, 4))
    np.testing.assert_array_equal((cov * np.float32(0.25) * np.float32(255)).astype(np.uint8), want_mask)
    assert (p2f >= 0).mean() > 0.5  # the plane-sized faces cover most of every view
    assert len(np.unique(p2f)) > 20


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_vertex_normals_bit_exact(amb_lib, seed):
    from actionmesh_b200 import ops

    v, f = _mesh(seed)
    got = ops.vertex_normals(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()).cpu().numpy()
    np.testing.assert_array_equal(got.view(np.int32), vertex_normals_ref(v, f).view(np.int32))


def test_indexed_mesh_bit_exact_and_deterministic(amb_lib):
    cams, focal = _cams()
    v, f = _mesh(3)
    a = _gpu_render(v, f, cams, focal, 64)
    b = _gpu_render(v, f, cams, focal, 64)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()
    want_p2f, _, want_rgb = render_ref(v, f, cams, focal, 64)
    np.testing.assert_array_equal(a[1], want_p2f)
    np.testing.assert_array_equal(a[2], want_rgb)


def _candidate_pairs(pv, faces, S, rows, cols, margin=3, bucket=16):
    """(sample, face) pairs where the face's projected box, widened by `margin` samples, holds the sample."""
    n2 = 2 * S
    tri = pv[faces]                                               # (F, 3, 3)
    # sample index of NDC x: (1 - x) S - 1/2
    ix = (1 - tri[..., 0].astype(np.float64)) * S - 0.5
    iy = (1 - tri[..., 1].astype(np.float64)) * S - 0.5
    c0, c1 = np.floor(ix.min(1)) - margin, np.ceil(ix.max(1)) + margin
    r0, r1 = np.floor(iy.min(1)) - margin, np.ceil(iy.max(1)) + margin
    assert (tri[..., 2] > 0).all() and ((c1 - c0) < 4 * bucket).all() and ((r1 - r0) < 4 * bucket).all()
    nb = (n2 + bucket - 1) // bucket
    b_c0, b_c1 = np.clip(c0 // bucket, 0, nb - 1).astype(int), np.clip(c1 // bucket, 0, nb - 1).astype(int)
    b_r0, b_r1 = np.clip(r0 // bucket, 0, nb - 1).astype(int), np.clip(r1 // bucket, 0, nb - 1).astype(int)
    fb, bb = [], []
    for dr in range(5):
        for dc in range(5):
            ok = (b_r0 + dr <= b_r1) & (b_c0 + dc <= b_c1)
            fb.append(np.nonzero(ok)[0])
            bb.append(((b_r0 + dr) * nb + b_c0 + dc)[ok])
    fb, bb = np.concatenate(fb), np.concatenate(bb)
    order = np.argsort(bb, kind="stable")
    fb, bb = fb[order], bb[order]
    start = np.searchsorted(bb, np.arange(nb * nb))
    end = np.searchsorted(bb, np.arange(nb * nb), side="right")
    sb = (rows // bucket) * nb + cols // bucket
    ps = np.repeat(np.arange(len(rows)), end[sb] - start[sb])
    pf = np.concatenate([fb[start[b]:end[b]] for b in sb])
    keep = (rows[ps] >= r0[pf]) & (rows[ps] <= r1[pf]) & (cols[ps] >= c0[pf]) & (cols[ps] <= c1[pf])
    return ps[keep], pf[keep]


def test_depth9_mesh_over_16_frames_at_sampled_pixels(amb_lib):
    import geometry_exact as gx
    import triposg_vae_ref as ref
    from actionmesh_b200 import ops
    from actionmesh_b200.render import B200MeshVisualizer
    from actionmesh_b200.triposg_vae import refine_octree
    from render_ref import project

    grid = refine_octree(gx.rippled_field, ref.BOUNDS, 9)
    gv, gf = ops.dual_marching_cubes(grid)
    del grid
    base = (gv.cpu().numpy().astype(np.float64) * (2.01 / 504) - 1.005)
    faces = gf.cpu().numpy()
    assert len(faces) > 1_500_000
    S, n_frames, K = 256, 16, 4096
    frames = []
    for k in range(n_frames):  # a smooth deformation: a twist about +Y growing with k, and a bob
        a = 0.03 * k * base[:, 1]
        x, z = base[:, 0] * np.cos(a) - base[:, 2] * np.sin(a), base[:, 0] * np.sin(a) + base[:, 2] * np.cos(a)
        frames.append(np.stack([x, base[:, 1] + 0.01 * k, z], 1).astype(np.float32))

    class M:
        def __init__(self, v):
            self.vertices, self.faces = v, faces

    vis = B200MeshVisualizer(image_size=S)
    grid_frames = vis.render_frames([M(v) for v in frames]).numpy()
    assert grid_frames.shape == (n_frames, S, 3 * S, 3)
    cams, focal = _cams()
    rng = np.random.default_rng(9)
    for k in (0, 7, 15):
        v = frames[k]
        normals = vertex_normals_ref(v, faces)
        ii, jj = rng.integers(0, S, (len(cams), K)), rng.integers(0, S, (len(cams), K))
        quads = []
        for c, cam in enumerate(cams):
            rows = np.concatenate([2 * ii[c], 2 * ii[c], 2 * ii[c] + 1, 2 * ii[c] + 1])
            cols = np.concatenate([2 * jj[c], 2 * jj[c] + 1, 2 * jj[c], 2 * jj[c] + 1])
            ps, pf = _candidate_pairs(project(v, cam, focal), faces, S, rows, cols)
            quads.append(rasterize_pairs_ref(v, faces, cam, focal, S, rows, cols, ps, pf).reshape(4, K).T)
        quad = np.stack(quads)
        assert (quad >= 0).mean() > 0.1 and (quad < 0).mean() > 0.5  # samples on and off the mesh
        mask, rgb = shade_ref(v, faces, normals, cams, focal, S, quad, ii, jj)
        for c in range(len(cams)):
            cell = grid_frames[k, :, c * S:(c + 1) * S]
            np.testing.assert_array_equal(cell[ii[c], jj[c]], rgb[c])
        # the mask at the samples: partial coverage shows as a composite between the normal colour and white
        assert {63, 127, 191} <= set(np.unique(mask).tolist())
    # pix_to_face itself at the sampled pixels of one frame
    vt, ft, ct = torch.from_numpy(frames[15]).cuda(), torch.from_numpy(faces).cuda(), torch.from_numpy(cams).cuda()
    p2f = ops.rasterize(vt, ft, ct, focal, S).cpu().numpy()
    np.testing.assert_array_equal(p2f[np.arange(len(cams))[:, None], 2 * ii, 2 * jj], quad[..., 0])


def test_visualizer_writes_the_grid_video(amb_lib, tmp_path):
    import cv2
    from PIL import Image

    from actionmesh_b200.render import B200MeshVisualizer

    class M:
        def __init__(self, v, f):
            self.vertices, self.faces = v, f

    v, f = _mesh(4, 200, 500)
    meshes = [M(v * (1 + 0.05 * k), f) for k in range(5)] + [M(np.zeros((0, 3)), np.zeros((0, 3), int))]
    S = 32
    frames = [Image.fromarray(np.full((40, 60, 4), 30 * k, np.uint8), "RGBA") for k in range(7)]
    vis = B200MeshVisualizer(image_size=S)
    for inputs, cols in ((frames, 4), (None, 3)):
        out = tmp_path / f"run{cols}"
        paths = vis.render(meshes, device="cuda", output_dir=str(out), input_frames=inputs)
        assert paths == [out / "grid_normal.mp4"] and paths[0].exists()
        cap = cv2.VideoCapture(str(paths[0]))
        n = 0
        while True:
            ok, fr = cap.read()
            if not ok:
                break
            assert fr.shape == (S, cols * S, 3)
            n += 1
        cap.release()
        assert n == len(meshes)
    grid = vis.render_frames(meshes, frames).numpy()
    assert (grid[-1, :, S:] == 255).all()  # the empty mesh gives white cells
    idx = [round(i * 6 / 5 + 1e-4) for i in range(6)]
    for k in range(6):  # input column: the reference's grid steps on the resampled frame (resize, paste, drop alpha)
        cell = Image.new("RGBA", (S, S), (0, 0, 0, 0))
        cell.paste(frames[idx[k]].resize((S, S)), (0, 0))
        np.testing.assert_array_equal(grid[k, :, :S], np.asarray(cell.convert("RGB")))
    assert vis.render([], output_dir=str(tmp_path / "none")) == []


def test_cpu_inputs_are_refused(amb_lib):
    from actionmesh_b200 import AmbError, ops
    from actionmesh_b200.render import B200MeshVisualizer

    cams, focal = _cams()
    v, f = _mesh(5, 50, 80)
    vt, ft, ct = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(cams).cuda()
    with pytest.raises(AmbError):
        ops.rasterize(vt, ft, ct.cpu(), focal, 8)
    with pytest.raises(AmbError):
        ops.vertex_normals(vt.cpu(), ft)
    p2f = ops.rasterize(vt, ft, ct, focal, 8)
    with pytest.raises(AmbError):
        ops.shade_normals(vt, ft, ops.vertex_normals(vt, ft), ct, focal, p2f.cpu())

    class M:
        vertices, faces = v, f

    with pytest.raises(AmbError):
        B200MeshVisualizer(image_size=8, device="cpu").render([M()], device="cpu", output_dir="unused", input_frames=None)


def test_launch_counts(amb_lib):
    from actionmesh_b200 import ops

    cams, focal = _cams()
    v, f = _mesh(6, 50, 80)
    vt, ft, ct = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(cams).cuda()
    n0 = ops.launch_count
    normals = ops.vertex_normals(vt, ft)
    assert ops.launch_count - n0 == 12
    n0 = ops.launch_count
    p2f = ops.rasterize(vt, ft, ct, focal, 16)
    assert ops.launch_count - n0 == 5
    n0 = ops.launch_count
    ops.shade_normals(vt, ft, normals, ct, focal, p2f)
    assert ops.launch_count - n0 == 1
    n0 = ops.launch_count
    ops.rasterize(vt, ft[:0], ct, focal, 16)
    assert ops.launch_count - n0 == 2
