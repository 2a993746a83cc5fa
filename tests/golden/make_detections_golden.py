"""Golden inputs for detector-fed streaming (push_detections), produced by the REAL reference.

    python tests/golden/make_detections_golden.py [--reference DIR]

Writes `tests/golden/detections/*.npz`.  Each case is a synthetic video as a 2-D detector leaves
it: a Detectron-format `.npz` (`boxes`, `keypoints`, `metadata`; one person in every detected frame,
empty lists in the frames without a detection, as inference/infer_video_d2.py writes them).  The
reference's own `data/prepare_data_2d_custom.decode` reads it back (one person per frame, the missed
frames filled by np.interp), and `common/camera.normalize_screen_coordinates` normalises the result
as run.py:96 applies it to every camera's keypoints.  Entries:
  kps_px  (T, 17, 2) float32  the detector's pixel keypoints, NaN in the frames without a detection
  mask    (T,) bool           frames with a detection
  xn      (T, 17, 2) float32  the reference's normalised keypoints (decode -> normalize)
  meta    json: T, w, h, seed
`make_case(name, reference_dir)` regenerates one case (used by the CPU test that checks the files).
"""
import argparse
import contextlib
import io
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "detections")

def _gaps_1_to_60(T, rng):
    """A leading gap of 5, interior gaps of every length 1..60 between runs of 1-2 detections,
    and a trailing gap of 7."""
    m = np.zeros(T, bool)
    t = 5
    for g in range(1, 61):
        run = 1 + int(g % 7 == 0)
        m[t:t + run] = True
        t += run + g
    m[t:T - 7] = True
    return m


def _random_gaps(T, rng):
    """Detections with miss probability 0.3 in geometric runs, a leading and a trailing gap."""
    m = np.ones(T, bool)
    t = 0
    while t < T:
        if rng.rand() < 0.3:
            g = int(rng.geometric(0.15))
            m[t:t + g] = False
            t += g
        t += int(rng.geometric(0.4))
    m[:3] = False
    m[-4:] = False
    m[T // 2] = True
    return m


def _single(T, rng):
    m = np.zeros(T, bool)
    m[17] = True
    return m


# name -> (frames, w, h, seed, mask builder)
CASES = {
    "gaps_1920x1080": (1930, 1920, 1080, 41, _gaps_1_to_60),
    "random_1000x1002": (400, 1000, 1002, 42, _random_gaps),
    "single_640x480": (40, 640, 480, 43, _single),
}


def make_video(name):
    """The detector's view of case `name`: (kps_px (T, 17, 2) with NaN where missed, mask, w, h)."""
    T, w, h, seed, builder = CASES[name]
    rng = np.random.RandomState(seed)
    mask = builder(T, rng)
    assert len(mask) == T and mask.any()
    # a person walking across the frame, with per-joint jitter: pixel coordinates in [0, w] x [0, h]
    base = np.stack([rng.uniform(0.2, 0.8, 17) * w, rng.uniform(0.2, 0.8, 17) * h], -1)
    drift = np.cumsum(rng.normal(0, 2.0, (T, 1, 2)), 0)
    kps = (base[None] + drift + rng.normal(0, 1.5, (T, 17, 2))).astype(np.float32)
    kps[~mask] = np.nan
    return kps, mask, w, h


def _detectron_npz(path, kps, mask, w, h, rng):
    """infer_video_d2.py's output format: per frame [[], boxes (n, 5)] and [[], [kp (4, 17)]]."""
    boxes, keypoints = [], []
    for t in range(len(mask)):
        if not mask[t]:
            boxes.append([[], []])
            keypoints.append([[], []])
            continue
        lo, hi = kps[t].min(0), kps[t].max(0)
        box = np.array([[lo[0], lo[1], hi[0], hi[1], rng.uniform(0.8, 1.0)]], np.float32)
        kp = np.zeros((4, 17), np.float32)
        kp[:2] = kps[t].T
        kp[2] = rng.uniform(1, 5, 17)
        kp[3] = rng.uniform(0.5, 1, 17)
        boxes.append([[], box])
        keypoints.append([[], [kp]])
    bb = np.empty(len(boxes), object)
    bb[:] = boxes
    kk = np.empty(len(keypoints), object)
    kk[:] = keypoints
    np.savez_compressed(path, boxes=bb, segments=[], keypoints=kk,
                        metadata={"w": w, "h": h})


def make_case(name, reference_dir):
    for d in (os.path.join(reference_dir, "data"), reference_dir):
        if d not in sys.path:
            sys.path.insert(0, d)
    from prepare_data_2d_custom import decode
    from common.camera import normalize_screen_coordinates
    T, w, h, seed, _ = CASES[name]
    kps, mask, w, h = make_video(name)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, name + ".npz")
        _detectron_npz(path, kps, mask, w, h, np.random.RandomState(seed + 1000))
        with contextlib.redirect_stdout(io.StringIO()):
            data, video_meta = decode(path)
    assert video_meta == {"w": w, "h": h}
    kp = data[0]["keypoints"].astype("float32")   # prepare_data_2d_custom.py: the stored array
    xn = kp.copy()
    xn[..., :2] = normalize_screen_coordinates(xn[..., :2], w=video_meta["w"], h=video_meta["h"])
    meta = dict(T=T, w=w, h=h, seed=seed)
    return {"kps_px": kps, "mask": mask, "xn": xn.astype(np.float32),
            "meta": np.array(json.dumps(meta))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=None)
    args = ap.parse_args()
    ref = args.reference
    if ref is None:
        sys.path.insert(0, ROOT)
        from oracle import stage_ref
        ref = stage_ref.reference_dir()
    if ref is None or not os.path.exists(os.path.join(ref, "data", "prepare_data_2d_custom.py")):
        raise SystemExit("no reference checkout with data/prepare_data_2d_custom.py: pass --reference")
    os.makedirs(OUT, exist_ok=True)
    for name in CASES:
        case = make_case(name, ref)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **case)
        print(f"{path}: T {len(case['mask'])}, {int((~case['mask']).sum())} missed, "
              f"{os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
