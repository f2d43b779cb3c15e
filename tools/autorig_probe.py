"""Time `autorig.fit_auto_rig` (default rounds and sweeps, 32 joints) on 31-frame animations with about 20 000 and 200 000
vertices: a host clock around each call, which ends in a device synchronise, one warm-up call, then the median of
--repeats calls.  Also reports the fit's RMS and maximum error next to the flat SSDR bones' RMS error (relative to the rest
bounding-box diagonal), the size of the written auto_rigged_mesh.glb, and the card and its power limit, read in the same
run.

The animation is tests/autorig_synthetic.py's skeleton (two tubes, seven segments turning by up to 60 degrees about their
pivots, a moving root, 50 / 50 skin weights on the rings at the horizontal tube's pivots), meshed finely enough for the
vertex counts; 32 joints over-segment its seven parts.

    python tools/autorig_probe.py [--repeats 3] [--out probe.json]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

SIZES = {20000: (0.01, 50), 200000: (0.003, 160)}     # vertices -> (ring step, vertices per ring)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--joints", type=int, default=32)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("autorig_probe: no CUDA device")
    import __graft_entry__ as ge

    ge.build()
    import autorig_synthetic as syn
    from actionmesh_b200 import autorig
    from actionmesh_b200.gltf import write_animated_glb, write_auto_rig_glb

    result = {"card": card(), "frames": 31, "joints": args.joints, "rounds": autorig.DEFAULT_ROUNDS,
              "sweeps": autorig.DEFAULT_SWEEPS, "sizes": []}
    for target, (step, around) in SIZES.items():
        rest, faces, W = syn.mesh(step=step, around=around)
        v, _ = syn.animate(rest, W, T=31)
        autorig.fit_auto_rig(v, faces, args.joints)
        times = []
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fit = autorig.fit_auto_rig(v, faces, args.joints)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        with tempfile.TemporaryDirectory() as tmp:
            write_auto_rig_glb(os.path.join(tmp, "a.glb"), fit, faces)
            write_animated_glb(os.path.join(tmp, "b.glb"), v, faces)
            sizes = [os.path.getsize(os.path.join(tmp, n)) for n in ("a.glb", "b.glb")]
        row = {"vertices": len(rest), "median_s": float(np.median(times)), "times_s": times, "rms_error": fit.rms_error,
               "max_error": fit.max_error, "ssdr_rms_error": fit.ssdr_rms_error, "auto_rig_glb_bytes": sizes[0],
               "animated_glb_bytes": sizes[1]}
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
