"""Time `skinning.fit_skinning` (default iterations) on 31-frame animations of 20 000 and 200 000 vertices with 32 bones: a host
clock around each call, which ends in a device synchronise, one warm-up call, then the median of --repeats calls.  Also
reports the fit's RMS and maximum error (relative to the rest bounding-box diagonal), the sizes of skinned_mesh.glb and
animated_mesh.glb for the same animation (2 V random faces), and the card and its power limit, read in the same run.

    python tools/skinning_probe.py [--repeats 5] [--out probe.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def animation(V: int, T: int = 31, seed: int = 0) -> np.ndarray:
    """(T, V, 3): points on a bumpy closed surface, twisted, bent and translated smoothly over the frames."""
    rng = np.random.default_rng(seed)
    d = rng.standard_normal((V, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rest = d * (1 + 0.2 * np.sin(3 * d[:, :1]) * np.cos(2 * d[:, 1:2])) * np.array([0.6, 0.6, 1.5])
    out = []
    for t in range(T):
        s = t / max(T - 1, 1)
        a = 0.8 * s * rest[:, 2:3]
        x = rest[:, :1] * np.cos(a) - rest[:, 1:2] * np.sin(a) + 0.3 * s * rest[:, 2:3] ** 2
        y = rest[:, :1] * np.sin(a) + rest[:, 1:2] * np.cos(a)
        out.append(np.concatenate([x, y, rest[:, 2:3]], 1) + np.array([0.1 * s, 0.0, 0.05 * np.sin(3 * s)]))
    return np.stack(out)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--bones", type=int, default=32)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("skinning_probe: no CUDA device")
    import __graft_entry__ as ge

    ge.build()
    from actionmesh_b200.gltf import write_animated_glb, write_skinned_glb
    from actionmesh_b200.skinning import fit_skinning

    result = {"card": card(), "frames": 31, "bones": args.bones, "sizes": []}
    for V in (20000, 200000):
        v = animation(V)
        fit_skinning(v, args.bones)
        times = []
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fit = fit_skinning(v, args.bones)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        faces = np.random.default_rng(1).integers(0, V, (2 * V, 3))
        with tempfile.TemporaryDirectory() as d:
            write_skinned_glb(os.path.join(d, "s.glb"), fit, faces)
            write_animated_glb(os.path.join(d, "a.glb"), v, faces)
            sizes = {"skinned_glb_bytes": os.path.getsize(os.path.join(d, "s.glb")),
                     "animated_glb_bytes": os.path.getsize(os.path.join(d, "a.glb"))}
        row = {"vertices": V, "median_s": float(np.median(times)), "times_s": times, "iterations": len(fit.history) - 1,
               "rms_error": fit.rms_error, "max_error": fit.max_error, **sizes}
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
