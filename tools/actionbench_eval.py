"""Score a directory of predicted animations with ActionBench's CD-3D, CD-4D and CD-M on the GPU.

    python tools/actionbench_eval.py --gt_root GT --pred_root PRED --output_csv results.csv

Restates actionbench/evaluate_dataset.py on `actionmesh_b200.evaluation.compute_chamfer_3d_4d`:
  * ground truth: {gt_root}/{uid}/surfaces.npy, (T, N, >= 3), of which [..., :3] as fp32;
  * prediction: {pred_root}/{uid}/mesh_*.glb in natural order, truncated to the T ground-truth frames;
  * the uids present on both sides are scored in sorted order; a failing uid gives a row with status "error" and its
    message, and the run goes on;
  * the CSV (columns uid, cd_3d, cd_4d, cd_motion, n_frames, status, error_message) and <csv stem>.summary.json are
    rewritten after every uid; a rerun keeps the rows that succeeded and retries the others (--recompute redoes all).
Loading .glb files needs trimesh, imported only when a mesh is loaded.  Meshes the pipeline produced can be scored
directly with compute_chamfer_3d_4d.
"""
from __future__ import annotations

import argparse
import csv
import json
import math
import os
import re
import sys
from pathlib import Path

import numpy as np

COLUMNS = ["uid", "cd_3d", "cd_4d", "cd_motion", "n_frames", "status", "error_message"]


def natural_sorted(names) -> list:
    """Sort by the digit runs of each name as numbers and the rest as lower-case text (natsort's default order on these
    file names)."""
    def key(name):
        parts = re.split(r"(\d+)", os.path.basename(str(name)))
        return [(0, int(p), "") if p.isdigit() else (1, 0, p.lower()) for p in parts if p != ""]
    return sorted(names, key=key)


def find_uids(gt_root: Path, pred_root: Path, mesh_pattern: str = "mesh_*.glb") -> list[str]:
    gt = {p.parent.name for p in gt_root.glob("*/surfaces.npy")}
    pred = {p.relative_to(pred_root).parts[0] for p in pred_root.glob(f"*/{mesh_pattern}")}
    if not gt:
        raise FileNotFoundError(f"No GT samples found in {gt_root}. Expected */surfaces.npy files.")
    if not pred:
        raise FileNotFoundError(f"No predictions found in {pred_root}. Expected */{mesh_pattern} files.")
    if not gt & pred:
        raise ValueError(f"No common UIDs between GT and predictions. GT UIDs: {len(gt)}, Pred UIDs: {len(pred)}.")
    for what, missing in (("predictions", gt - pred), ("GT", pred - gt)):
        if missing:
            print(f"warning: missing {what} for {len(missing)} uids", file=sys.stderr)
    return sorted(gt & pred)


def load_meshes(paths: list) -> list:
    try:
        import trimesh
    except ImportError as exc:
        raise RuntimeError("loading .glb predictions needs trimesh (pip install trimesh); meshes already in memory can be "
                           "scored with actionmesh_b200.evaluation.compute_chamfer_3d_4d") from exc
    return [trimesh.load(p, force="mesh") for p in paths]


def default_scorer(device="cuda", n_pts_icp=10_000, n_pts_chamfer=100_000, seed=44, is_4d=True):
    def score(gt_pc: np.ndarray, mesh_paths: list) -> tuple[float, float, float]:
        from actionmesh_b200.evaluation import compute_chamfer_3d_4d

        return compute_chamfer_3d_4d(gt_pc, load_meshes(mesh_paths), device=device, is_4D=is_4d, n_pts_icp=n_pts_icp,
                                     n_pts_chamfer=n_pts_chamfer, seed=seed)
    return score


def evaluate_sample(uid: str, gt_root: Path, pred_root: Path, scorer, mesh_pattern: str = "mesh_*.glb") -> dict:
    row = {"uid": uid, "cd_3d": math.nan, "cd_4d": math.nan, "cd_motion": math.nan, "n_frames": 0, "status": "error",
           "error_message": ""}
    try:
        gt_path, pred_dir = gt_root / uid / "surfaces.npy", pred_root / uid
        if not gt_path.exists():
            row["error_message"] = f"GT not found: {gt_path}"
            return row
        if not pred_dir.exists():
            row["error_message"] = f"Pred dir not found: {pred_dir}"
            return row
        gt_pc = np.ascontiguousarray(np.load(gt_path)[..., :3], dtype=np.float32)
        row["n_frames"] = n = gt_pc.shape[0]
        paths = natural_sorted(pred_dir.glob(mesh_pattern))
        if not paths:
            raise FileNotFoundError(f"No mesh files found in {pred_dir}")
        if len(paths) < n:
            raise ValueError(f"Not enough meshes: found {len(paths)}, need {n}")
        row["cd_3d"], row["cd_4d"], row["cd_motion"] = (float(v) for v in scorer(gt_pc, [str(p) for p in paths[:n]]))
        row["status"] = "success"
    except Exception as exc:  # noqa: BLE001 — one failing uid must not stop the dataset
        row["status"], row["error_message"] = "error", str(exc)
        print(f"[{uid}] Error: {exc}", file=sys.stderr)
    return row


def summary(rows: list[dict]) -> dict:
    ok = [r for r in rows if r["status"] == "success"]
    out = {"n_total": len(rows), "n_success": len(ok), "n_failed": len(rows) - len(ok),
           "success_rate": len(ok) / len(rows) if rows else 0.0}
    for k in ("cd_3d", "cd_4d", "cd_motion"):
        out[f"{k}_mean"] = float(np.mean([r[k] for r in ok])) if ok else math.nan
    return out


def load_existing(path: Path) -> dict[str, dict]:
    if not path.exists():
        return {}
    rows = {}
    with open(path, newline="") as f:
        for r in csv.DictReader(f):
            for k in ("cd_3d", "cd_4d", "cd_motion"):
                r[k] = float(r[k])
            r["n_frames"] = int(r["n_frames"])
            rows[r["uid"]] = r
    return rows


def save(rows: list[dict], path: Path) -> None:
    path.parent.mkdir(parents=True, exist_ok=True)
    with open(path, "w", newline="") as f:
        w = csv.DictWriter(f, fieldnames=COLUMNS)
        w.writeheader()
        w.writerows(rows)
    with open(path.with_suffix(".summary.json"), "w") as f:
        json.dump(summary(rows), f, indent=2)


def evaluate_dataset(gt_root: str, pred_root: str, output_csv: str | None = None, scorer=None,
                     mesh_pattern: str = "mesh_*.glb", recompute: bool = False, **score_args) -> list[dict]:
    gt_root, pred_root = Path(gt_root), Path(pred_root)
    out = Path(output_csv) if output_csv else None
    scorer = scorer or default_scorer(**score_args)
    existing = load_existing(out) if out and not recompute else {}
    rows = []
    for uid in find_uids(gt_root, pred_root, mesh_pattern):
        prev = existing.get(uid)
        if prev is not None and prev["status"] == "success":
            rows.append(prev)
            continue
        rows.append(evaluate_sample(uid, gt_root, pred_root, scorer, mesh_pattern))
        r = rows[-1]
        if r["status"] == "success":
            print(f"[{uid}] CD_3D={r['cd_3d']:.3f}, CD_4D={r['cd_4d']:.3f}, CD_Motion={r['cd_motion']:.3f}")
        if out:
            save(rows, out)
    if out:
        save(rows, out)
    return rows


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--gt_root", required=True)
    ap.add_argument("--pred_root", required=True)
    ap.add_argument("--output_csv", default=None)
    ap.add_argument("--device", default="cuda")
    ap.add_argument("--n_pts_icp", type=int, default=10_000)
    ap.add_argument("--n_pts_chamfer", type=int, default=100_000)
    ap.add_argument("--seed", type=int, default=44)
    ap.add_argument("--mesh_pattern", default="mesh_*.glb")
    ap.add_argument("--recompute", action="store_true")
    ap.add_argument("--no_4d", action="store_true", help="skip the motion Chamfer distance (cd_motion = 0)")
    a = ap.parse_args()
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    rows = evaluate_dataset(a.gt_root, a.pred_root, a.output_csv, mesh_pattern=a.mesh_pattern, recompute=a.recompute,
                            device=a.device, n_pts_icp=a.n_pts_icp, n_pts_chamfer=a.n_pts_chamfer, seed=a.seed,
                            is_4d=not a.no_4d)
    print(json.dumps(summary(rows), indent=2))


if __name__ == "__main__":
    main()
