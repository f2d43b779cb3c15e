"""Time background removal on one GPU: ms per frame of B200BackgroundRemover at a 1024 x 1024 model input, against the fp32
restatement of the reference (tests/rmbg_ref.py) in PyTorch eager on the same GPU with cuDNN TF32 on (the reference's
default) and off, plus a per-kernel CUDA-event breakdown and the shape arithmetic of the convolutions.

    python tools/rmbg_bench.py [--frames 10] [--warmup 2] [--out DIR]

Weights are the tests' seeded synthetic ones (the time does not depend on their values).  Prints one JSON line, with the
card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def conv_flops(size=(1024, 1024)) -> dict:
    """FLOPs of every convolution at a model input size: real (2 * 9 * C_in * C_out per output pixel), padded to the GEMM's
    N and K granularity, and the MMA work of the three-term split operand (3x the padded K)."""
    from actionmesh_b200 import ops
    from actionmesh_b200.background_removal import DECODER, ENCODER, rsu_convs

    pad = lambda n: (n + 63) // 64 * 64
    real = padded = 0
    h, w = ops.conv3x3_out(size[0], 2, 1, 1), ops.conv3x3_out(size[1], 2, 1, 1)
    real += 2 * h * w * 27 * 64
    padded += 2 * h * w * 64 * 64
    sizes = [(h, w)]
    for _ in ENCODER[1:]:
        sizes.append(((sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2))
    for (stage, depth, cin, mid, cout), (sh, sw) in list(zip(ENCODER, sizes)) + list(zip(DECODER, sizes[-2::-1])):
        levels = [(sh, sw)]
        for _ in range(max(depth - 2, 0)):
            levels.append(((levels[-1][0] + 1) // 2, (levels[-1][1] + 1) // 2))
        for name, i, o, _ in rsu_convs(depth, cin, mid, cout):
            lvl = 0 if depth == 0 or name in ("rebnconvin", "rebnconv1", "rebnconv1d") else \
                min(int(name[8:].rstrip("d")) - 1, depth - 2)
            ph, pw = levels[lvl]
            real += 2 * ph * pw * 9 * i * o
            padded += 2 * ph * pw * pad(9 * i) * pad(o)
    return dict(real=real, padded=padded, split=3 * padded)


def _gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except (OSError, IndexError, ValueError, subprocess.TimeoutExpired):
        return dict(gpu=torch.cuda.get_device_name(), power_limit="unknown", max_sm_clock="unknown")


def _time(fn, frames: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(frames):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / frames


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rmbg_bench needs a CUDA device")
    import rmbg_ref
    from actionmesh_b200 import ops
    from actionmesh_b200.background_removal import B200BackgroundRemover

    size = (1024, 1024)
    sd = rmbg_ref.make_state_dict(0)
    m = B200BackgroundRemover(model_input_size=size).to("cuda")
    m.load_state_dict(sd)
    image = rmbg_ref.synthetic_frame(1080, 1920, 7)
    rgb = torch.from_numpy(image).cuda()
    res = dict(model_input=list(size), frame=list(image.shape[:2]), **_gpu_info())
    res["b200_ms_per_frame"] = _time(lambda: m._run(rgb), args.frames, args.warmup)
    res["b200_forward_ms_per_frame"] = _time(lambda: m.forward(image), args.frames, 1)   # with the host copies

    # per-kernel breakdown of one frame
    ops.event_tags = {"rmbg_resize", "rmbg_im2col", "rmbg_conv", "rmbg_pool", "rmbg_upsample", "rmbg_mask_head", "rmbg_refine"}
    ops.event_log = []
    m._run(rgb)
    torch.cuda.synchronize()
    breakdown = {}
    for tag, e0, e1, _ in ops.event_log:
        breakdown[tag] = breakdown.get(tag, 0.0) + e0.elapsed_time(e1)
    ops.event_log, ops.event_tags = None, set()
    res["breakdown_ms"] = {k: round(v, 3) for k, v in sorted(breakdown.items(), key=lambda kv: -kv[1])}

    x = rmbg_ref.preprocess(image, size, "cuda")
    sd_cuda = {k: v.cuda() for k, v in sd.items()}
    for tf32 in (True, False):
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
        with torch.no_grad():
            ms = _time(lambda: rmbg_ref.rmbg_forward(sd_cuda, x), args.frames, args.warmup)
        res[f"oracle_eager_{'tf32' if tf32 else 'fp32'}_ms_per_frame"] = ms
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = False
    f = conv_flops(size)
    res["conv_gflop"] = {k: round(v / 1e9, 1) for k, v in f.items()}
    conv_ms = breakdown.get("rmbg_conv", 0.0)
    if conv_ms:
        res["conv_gemm_tflops_split"] = round(f["split"] / conv_ms / 1e9, 1)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "rmbg_bench.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
