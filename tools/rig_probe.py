"""Time `rig.fit_rig_animation` (default sweeps) on 31-frame animations of a 65-joint rig with 20 000 and 200 000 vertices: a
host clock around each call, which ends in a device synchronise, one warm-up call, then the median of --repeats calls.
Also reports the fit's RMS and maximum error (relative to the rest bounding-box diagonal) and the card and its power
limit, read in the same run.

The rig: a root with five chains of 13 joints (64 joints below the root, depth 14), every vertex near a bone and
weighted to its joint and, for two vertices in three, the joint's parent.  The animation is the rig's own forward
kinematics (tests/rig_ref.py) with every local rotation turned by up to 30 degrees and a moving root, so an exact fit
exists.

    python tools/rig_probe.py [--repeats 3] [--out probe.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def axis_angle(axis, ang) -> np.ndarray:
    axis = np.asarray(axis, float) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def rig_and_animation(V: int, T: int = 31, seed: int = 0):
    from actionmesh_b200 import rig as rigmod
    from actionmesh_b200.gltf import _quaternions
    import rig_ref

    rng = np.random.default_rng(seed)
    parent, offset = [-1], [np.zeros(3)]
    for c in range(5):
        d = np.array([np.cos(2 * np.pi * c / 5), 1.0, np.sin(2 * np.pi * c / 5)]) * 0.15
        for k in range(13):
            parent.append(0 if k == 0 else len(parent) - 1)
            offset.append(d)
    J = len(parent)
    q0 = _quaternions(np.stack([axis_angle(rng.standard_normal(3), rng.uniform(0, 0.2)) for _ in range(J)]))
    G0 = np.zeros((J, 4, 4))
    for j in range(J):
        loc = np.eye(4)
        loc[:3, :3] = rigmod._rotation_matrix(q0[j])
        loc[:3, 3] = offset[j]
        G0[j] = (G0[parent[j]] if parent[j] >= 0 else np.eye(4)) @ loc
    heads = G0[:, :3, 3]
    pick = rng.integers(1, J, V)
    pts = heads[pick] + rng.uniform(0, 1, (V, 1)) * (heads[np.array(parent)[pick]] - heads[pick]) \
        + 0.02 * rng.standard_normal((V, 3))
    sb, sw = np.zeros((V, 8), np.int32), np.zeros((V, 8))
    sb[:, 0], sb[:, 1] = pick, np.array(parent)[pick]
    w = rng.uniform(0.3, 1, (V, 2))
    w[np.arange(V) % 3 == 0, 1] = 0
    sw[:, :2] = w / w.sum(1, keepdims=True)
    rig = SimpleNamespace(order=np.arange(J), parent=np.array(parent), scale=np.ones((J, 3)), above=np.tile(np.eye(4), (J, 1, 1)),
                          binds=np.linalg.inv(G0), bind_joint=np.arange(J), rotation=q0, translation=np.array(offset),
                          points=pts, rest=pts.copy(), slot_bind=sb, slot_weight=sw)
    a = rigmod.rig_arrays(rig)
    rots = np.zeros((T, J, 9))
    trs = np.ascontiguousarray(np.broadcast_to(a.translations, (T, J, 3))).copy()
    for t in range(T):
        for j in range(J):
            rots[t, j] = (a.rotations[j].reshape(3, 3) @ axis_angle(rng.standard_normal(3),
                                                                   np.deg2rad(rng.uniform(0, 30)))).ravel()
        trs[t, 0] = 0.2 * rng.standard_normal(3)
    return rig, rig_ref.posed(a, rots, trs)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("rig_probe: no CUDA device")
    import __graft_entry__ as ge

    ge.build()
    from actionmesh_b200.rig import DEFAULT_SWEEPS, fit_rig_animation

    result = {"card": card(), "frames": 31, "joints": 65, "sweeps": DEFAULT_SWEEPS, "sizes": []}
    for V in (20000, 200000):
        rig, v = rig_and_animation(V)
        fit_rig_animation(rig, v)
        times = []
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fit = fit_rig_animation(rig, v)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        row = {"vertices": V, "median_s": float(np.median(times)), "times_s": times, "rms_error": fit.rms_error,
               "max_error": fit.max_error}
        print(json.dumps(row), flush=True)
        result["sizes"].append(row)
    result["card_after"] = card()
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
