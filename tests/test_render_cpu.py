"""Normal renderer checks that need no GPU: the cameras against their closed form, known answers of the float32
restatement (tests/render_ref.py), the input-frame resampling, the mp4 writer, host validation and the C ABI's argument
checks (fake pointers, no launch)."""
import math

import numpy as np
import pytest

from render_ref import camera_table, project, rasterize_ref, render_ref, sample_ndc, vertex_normals_ref

F = 2.1875


def _cams(tags=("U000", "U004", "U008")):
    from actionmesh_b200.render import uniform_cameras

    cams = uniform_cameras()
    return camera_table({t: cams[t] for t in tags})


def _from_view(points_view: np.ndarray, cam: np.ndarray) -> np.ndarray:
    """World points whose view-space coordinates are (approximately) points_view: X = (X_view - T) R^T, in float64."""
    R, T = cam[:9].reshape(3, 3).astype(np.float64), cam[9:12].astype(np.float64)
    return ((points_view - T) @ R.T).astype(np.float32)


def test_uniform_cameras_match_closed_form():
    from actionmesh_b200.render import uniform_cameras

    cams = uniform_cameras(distance=3.0)
    assert list(cams) == [f"U{i:03d}" for i in range(16)]
    for i, (tag, (R, T, f)) in enumerate(cams.items()):
        assert R.dtype == T.dtype == np.float32 and f == 2.1875
        th, ph = math.radians(i / 16 * 360), math.radians([70, 55, 85, 40][i % 4])
        C = 3.0 * np.array([math.sin(ph) * math.cos(th), math.cos(ph), -math.sin(ph) * math.sin(th)])
        z = -C / np.linalg.norm(C)
        x = np.cross([0.0, 1.0, 0.0], z)
        x /= np.linalg.norm(x)
        y = np.cross(z, x)
        Rw = np.stack([x, y, z], axis=1)
        np.testing.assert_allclose(R, Rw, atol=1e-6)
        np.testing.assert_allclose(T, -C @ Rw, atol=1e-6)
        np.testing.assert_allclose(-T.astype(np.float64) @ R.T.astype(np.float64), C, atol=1e-6)  # the centre back
    for tag in ("U000", "U004", "U008"):  # the visualizer's cameras all sit at 70 degrees
        R, T, _ = cams[tag]
        centre = -T.astype(np.float64) @ R.T.astype(np.float64)
        assert math.isclose(math.degrees(math.acos(centre[1] / 3.0)), 70.0, abs_tol=1e-4)


def test_square_covers_exactly_the_samples_strictly_inside():
    cams, f = _cams(("U000",))
    S = 16
    # NDC half-width between two sample rows, and a shift of an eighth of a sample in x so that no sample centre lies on the
    # shared diagonal either
    a, d = (0.5 + 0.25 / S) * 3.0 / F, 0.125 / S * 3.0 / F
    corners = _from_view(np.array([[d - a, -a, 3.0], [d + a, -a, 3.0], [d + a, a, 3.0], [d - a, a, 3.0]]), cams[0])
    faces = np.array([[0, 1, 2], [0, 2, 3]], dtype=np.int32)
    p2f = rasterize_ref(corners, faces, cams, f, S)[0]
    pv = project(corners, cams[0], f)
    lo_x, hi_x, lo_y, hi_y = pv[:, 0].min(), pv[:, 0].max(), pv[:, 1].min(), pv[:, 1].max()
    xs, ys = sample_ndc(np.arange(2 * S), 2 * S), sample_ndc(np.arange(2 * S), 2 * S)
    want = (ys[:, None] > lo_y) & (ys[:, None] < hi_y) & (xs[None, :] > lo_x) & (xs[None, :] < hi_x)
    assert want.sum() == (2 * S // 2) ** 2
    np.testing.assert_array_equal(p2f >= 0, want)


def _tri(cam, depth, scale=0.4, shift=(0.0, 0.0)):
    d = np.array([[-scale, -scale, 0.0], [scale, -scale, 0.0], [0.0, scale, 0.0]]) * depth / 3.0
    return _from_view(d + np.array([shift[0] * depth / 3, shift[1] * depth / 3, depth]), cam)


def test_nearer_triangle_wins_and_ties_go_to_the_lower_index():
    cams, f = _cams(("U000",))
    far, near = _tri(cams[0], 3.5), _tri(cams[0], 2.5, shift=(0.1, 0.0))
    verts = np.concatenate([far, near, near])
    faces = np.array([[0, 1, 2], [3, 4, 5], [6, 7, 8]], dtype=np.int32)
    p2f = rasterize_ref(verts, faces, cams, f, 16)[0]
    assert (p2f == 1).sum() > 0 and not (p2f == 2).any()  # face 2 repeats face 1 at the same depth: the lower index wins
    assert (p2f == 0).sum() > 0  # the far face shows where the near one does not cover it
    alone = rasterize_ref(far, faces[:1], cams, f, 16)[0]
    assert ((alone == 0) & (p2f == 1)).sum() > 0  # where both cover a sample, the nearer (1) is kept


def test_zero_area_and_behind_camera_faces_never_appear():
    cams, f = _cams(("U000",))
    tri = _tri(cams[0], 3.0, scale=0.8)
    flat = _from_view(np.array([[-0.5, 0.0, 3.0], [0.0, 0.0, 3.0], [0.5, 0.0, 3.0]]), cams[0])  # collinear
    behind = _from_view(np.array([[-1.0, -1.0, -2.0], [1.0, -1.0, -2.0], [0.0, 1.0, -2.0]]), cams[0])
    verts = np.concatenate([flat, behind, tri])
    faces = np.array([[0, 1, 2], [3, 4, 5], [6, 7, 8]], dtype=np.int32)
    p2f = rasterize_ref(verts, faces, cams, f, 16)
    assert not np.isin(p2f, [0, 1]).any() and (p2f == 2).any()


def _sphere(n_lat=24, n_lon=48, r=0.6):
    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    v = [[0, r, 0]] + [[r * np.sin(t) * np.cos(p), r * np.cos(t), r * np.sin(t) * np.sin(p)] for t in th for p in ph]
    v.append([0, -r, 0])
    faces = []
    ring = lambda i, j: 1 + i * n_lon + j % n_lon
    for j in range(n_lon):
        faces.append([0, ring(0, j + 1), ring(0, j)])
        faces.append([len(v) - 1, ring(n_lat - 2, j), ring(n_lat - 2, j + 1)])
    for i in range(n_lat - 2):
        for j in range(n_lon):
            faces += [[ring(i, j), ring(i, j + 1), ring(i + 1, j)], [ring(i, j + 1), ring(i + 1, j + 1), ring(i + 1, j)]]
    return np.array(v, dtype=np.float32), np.array(faces, dtype=np.int32)


def test_mask_levels_and_sphere_centre_colour():
    cams, f = _cams()
    verts, faces = _sphere()
    S = 24
    p2f, mask, rgb = render_ref(verts, faces, cams, f, S)
    assert set(np.unique(mask)) <= {0, 63, 127, 191, 255} and {0, 255} <= set(np.unique(mask))
    assert len(set(np.unique(mask))) > 2  # the silhouette has partial coverage
    xf = 1 - (2 * S + 1) / (2 * S)  # sample (2i, 2j) of the centre pixel i = j = S / 2
    for c, cam in enumerate(cams):
        # the exact sphere's normal where the sample's ray meets it, mapped as a point by the camera with T halved
        R, T = cam[:9].reshape(3, 3).astype(np.float64), cam[9:12].astype(np.float64)
        centre, ray = -T @ R.T, np.array([xf / f, xf / f, 1.0]) @ R.T
        ray /= np.linalg.norm(ray)
        t = -(centre @ ray) - math.sqrt((centre @ ray) ** 2 - centre @ centre + 0.6 ** 2)
        n = (centre + t * ray) / 0.6
        m = n @ R + T / 2
        want = np.floor(255 * (m / np.linalg.norm(m) + 1) / 2)
        assert abs(want - [127, 127, 255]).max() > 5  # the halved translation does change the colour
        np.testing.assert_allclose(rgb[c, S // 2, S // 2].astype(int), want, atol=2)
        assert (rgb[c][mask[c] == 0] == 255).all()  # background is white
    n = vertex_normals_ref(verts, faces)
    assert ((n * verts).sum(axis=1) / 0.6 > 0.999).all()  # outward and close to radial
    np.testing.assert_allclose(np.linalg.norm(n, axis=1), 1.0, atol=1e-6)


def test_resample_list_indices():
    from actionmesh_b200.render import resample_list

    assert resample_list(list(range(31)), 16) == [round(i * 30 / 15 + 1e-4) for i in range(16)]
    assert resample_list(list(range(10)), 4) == [0, 3, 6, 9]
    assert resample_list(list(range(3)), 5) == [0, 1, 1, 2, 2]  # 0.5 and 1.5 pushed up by the 1e-4
    assert resample_list([7, 8], 1) == [7] and resample_list([], 3) == [] and resample_list([1], 0) == []


def test_mp4_round_trip(tmp_path):
    """mp4v is lossy: the frame count and size survive exactly; a smooth synthetic grid comes back within a mean absolute
    difference of 8 levels (of 255)."""
    import cv2

    from actionmesh_b200.render import write_video

    n, h, w = 5, 64, 192
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    frames = np.stack([np.stack([(xx + 9 * k) % 256, yy * 4 % 256, np.full_like(xx, 40 * k)], -1) for k in range(n)])
    frames = frames.astype(np.uint8)
    path = tmp_path / "grid_normal.mp4"
    write_video(frames, path)
    cap = cv2.VideoCapture(str(path))
    got = []
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        got.append(fr[..., ::-1])
    cap.release()
    assert len(got) == n and got[0].shape == (h, w, 3)
    assert np.abs(np.stack(got).astype(float) - frames).mean() < 8.0


class _M:
    def __init__(self, v, f):
        self.vertices, self.faces = v, f


def test_host_validation():
    from actionmesh_b200.render import mesh_arrays

    v = np.zeros((3, 3))
    with pytest.raises(ValueError, match="face indices"):
        mesh_arrays(_M(v, [[0, 1, 3]]))
    with pytest.raises(ValueError, match="face indices"):
        mesh_arrays(_M(v, [[0, -1, 2]]))
    with pytest.raises(ValueError, match="non-finite"):
        mesh_arrays(_M(np.array([[0, 0, np.nan], [0, 0, 0], [1, 0, 0]]), [[0, 1, 2]]))
    with pytest.raises(ValueError, match="non-finite"):
        mesh_arrays(_M(np.array([[0, 0, 1e39], [0, 0, 0], [1, 0, 0]]), [[0, 1, 2]]))  # overflows float32
    verts, faces = mesh_arrays(_M(v, [[0, 1, 2], [0, 0, 1], [2, 1, 2], [2, 1, 0]]))
    assert verts.dtype == np.float32 and faces.dtype == np.int32
    np.testing.assert_array_equal(faces, [[0, 1, 2], [2, 1, 0]])  # faces that repeat a corner are dropped
    assert mesh_arrays(_M(np.zeros((0, 3)), np.zeros((0, 3))))[1].shape == (0, 3)


def test_visualizer_refuses_cpu():
    from actionmesh_b200 import AmbError
    from actionmesh_b200.render import B200MeshVisualizer

    with pytest.raises(AmbError):
        B200MeshVisualizer(image_size=8, device="cpu").render_frames([_M(np.eye(3), [[0, 1, 2]])])


def test_ops_refuse_cpu_tensors():
    import torch

    from actionmesh_b200 import AmbError, ops

    v, f = torch.eye(3), torch.tensor([[0, 1, 2]], dtype=torch.int32)
    with pytest.raises(AmbError):
        ops.vertex_normals(v, f)
    with pytest.raises(AmbError):
        ops.rasterize(v, f, torch.zeros(1, 12), F, 8)
    with pytest.raises(AmbError):
        ops.shade_normals(v, f, v, torch.zeros(1, 12), F, torch.zeros(1, 16, 16, dtype=torch.int32))


def test_render_abi_argument_validation(amb_lib):
    """The render entry points validate their arguments before any launch (fake non-null pointers)."""
    P = 16
    err = lambda: amb_lib.amb_last_error().decode()
    assert amb_lib.amb_render_vertex_normals(None, 3, P, P, P, P, None) < 0 and "null pointer" in err()
    assert amb_lib.amb_render_vertex_normals(P, -1, P, P, P, P, None) < 0 and "bad vertex count" in err()
    ras = lambda **k: amb_lib.amb_render_rasterize(k.get("v", P), k.get("nv", 3), P, k.get("nf", 1), P, k.get("c", 3), F,
                                                   k.get("s", 8), P, P, k.get("out", P), None)
    assert ras(out=None) < 0 and "null pointer" in err()
    assert ras(v=None) < 0 and "null pointer" in err()
    assert ras(v=None, c=0, nf=0) < 0 and "n_cameras >= 1" in err()  # no faces: the mesh pointers may be NULL
    assert ras(c=0) < 0 and "n_cameras >= 1" in err()
    assert ras(s=0) < 0 and "image_size >= 1" in err()
    assert ras(s=1 << 14) < 0 and "overflow" in err()               # 3 x 32768^2 samples
    assert ras(c=7, nf=357_000_000) < 0 and "overflow" in err()      # 7 x F queue entries
    assert ras(nf=1 << 29) < 0 and "bad mesh size" in err()         # 6 F
    assert ras(nv=-1) < 0 and "bad mesh size" in err()
    sh = lambda **k: amb_lib.amb_render_shade_normals(P, 3, P, 1, P, P, k.get("c", 3), F, k.get("s", 8), P,
                                                      k.get("out", P), k.get("row", 72), k.get("view", 24), None)
    assert sh(out=None) < 0 and "null pointer" in err()
    assert sh(c=0) < 0 and "n_cameras >= 1" in err()
    assert sh(s=0) < 0 and "image_size >= 1" in err()
    assert sh(s=1 << 14) < 0 and "overflow" in err()
    assert sh(row=23) < 0 and "bad strides" in err()
    assert sh(view=23) < 0 and "bad strides" in err()
