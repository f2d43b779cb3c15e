"""Regenerate tests/golden/rmbg_tiny.pt from the reference's OWN BriaRMBG and refinement.

    ACTIONMESH_REFERENCE=/path/to/actionmesh python tools/gen_rmbg_golden.py

Needs a checkout of facebookresearch/actionmesh: third_party/TripoSG/scripts/briarmbg.py is imported unchanged and run on
the CPU in fp32 with tests/rmbg_ref.make_state_dict(SEED) (seeded weights, RMS-calibrated BatchNorm statistics; no
weights are stored).  The frame is rmbg_ref.synthetic_frame(FRAME, FRAME_SEED) at model input size MODEL_SIZE, an odd,
non-square size: the pooling chain 100 x 132 -> ... -> 4 x 5 has partial ceil-mode windows and the decoder upsamples by
ratios other than 2.  Stored: sigmoid(d1) at the model size, the uint8 mask of _postprocess_mask and refine_mask's result
(cv2 Otsu; the reference's scikit-image labelling is replaced by scipy.ndimage.label with a 3x3 structure, which is
skimage.measure.label's documented 2-D default).
"""
from __future__ import annotations

import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import reference_loader  # noqa: E402
import rmbg_ref  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "rmbg_tiny.pt")
SEED = 0
FRAME, FRAME_SEED = (180, 240), 7
MODEL_SIZE = (200, 264)
MIN_SIZE = 200


def main() -> None:
    path = os.path.join(reference_loader.REFERENCE_ROOT, "third_party", "TripoSG", "scripts", "briarmbg.py")
    spec = importlib.util.spec_from_file_location("briarmbg", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    torch.manual_seed(0)
    net = mod.BriaRMBG().eval()
    net.load_state_dict(rmbg_ref.make_state_dict(SEED), strict=True)
    image = rmbg_ref.synthetic_frame(*FRAME, FRAME_SEED)
    with torch.no_grad():
        soft = net(rmbg_ref.preprocess(image, MODEL_SIZE))[0][0]
    mask = rmbg_ref.postprocess_mask(soft, image.shape[:2])
    refined = rmbg_ref.refine_mask(mask, MIN_SIZE)
    torch.save(dict(seed=SEED, frame=FRAME, frame_seed=FRAME_SEED, model_size=MODEL_SIZE, min_size=MIN_SIZE,
                    soft=soft[0, 0].clone(), mask=torch.from_numpy(mask.copy()), refined=torch.from_numpy(refined.copy())),
               GOLDEN)
    print(f"wrote {GOLDEN}: soft in [{soft.min():.4f}, {soft.max():.4f}], refined foreground {int((refined > 0).sum())} px")


if __name__ == "__main__":
    main()
