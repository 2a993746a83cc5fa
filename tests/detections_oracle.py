"""Host oracles for detector-fed streaming (StreamingSession.push_detections).

reference_sequence: what the reference's in-the-wild pipeline feeds the network for one video --
decode's np.interp over the frames without a detection (data/prepare_data_2d_custom.py:39-49),
then run.py:96's normalize_screen_coordinates -- or, with max_gap = G, the sequence the G rule
gives (the first L - G frames of a longer gap held at the detection before it).
pack_restated: a float64 numpy restatement of vp3d_stream_pack_detections, record by record.
"""
import numpy as np


def normalize(kp, w, h):
    """common/camera.py:14-18 as run.py:96 applies it: X / w * 2 - [1, h / w] into float32."""
    out = np.array(kp, np.float32, copy=True)
    out[..., :2] = out[..., :2] / w * 2 - [1, h / w]
    return out


def interpolated(kps_px, mask):
    """decode's fill: np.interp per joint and coordinate, stored as float32."""
    T = len(mask)
    idx = np.arange(T)
    kp = np.empty(kps_px.shape, np.float32)
    for j in range(kps_px.shape[1]):
        for c in range(2):
            kp[:, j, c] = np.interp(idx, idx[mask], kps_px[mask, j, c])
    return kp


def reference_sequence(kps_px, mask, w, h, max_gap=None):
    """The (T, J, 2) float32 normalised sequence of a video with at least one detection."""
    mask = np.asarray(mask, bool)
    kp = interpolated(kps_px, mask)
    if max_gap is not None:
        det = np.nonzero(mask)[0]
        for a, b in zip(det[:-1], det[1:]):
            for t in range(a + 1, b):
                if b - t > max_gap:
                    kp[t] = kps_px[a]
    return normalize(kp, w, h)


def _interp(l, r, num, den):
    slope = (r.astype(np.float64) - l.astype(np.float64)) / np.float64(den)
    return (slope * np.float64(num) + l.astype(np.float64)).astype(np.float32)


def _normalise(v, w, h):
    q = (v[..., 0:1] / np.float32(w)) * np.float32(2)
    p = (v[..., 1:2] / np.float32(w)) * np.float32(2)
    x = (q.astype(np.float64) - 1.0).astype(np.float32)
    y = (p.astype(np.float64) - np.float64(h) / np.float64(w)).astype(np.float32)
    return np.concatenate([x, y], -1)


def pack_restated(kps, slots, records, last):
    """vp3d_stream_pack_detections on the host: kps (S, k, J, 2) float32, slots (S, 3), records
    (rows, 5), last (S, J, 2) the stored detections; returns (out (rows, J, 2), new last)."""
    S, k, J, _ = kps.shape
    out = np.zeros((len(records), J, 2), np.float32)
    for r, (s, left, right, num, den) in enumerate(records):
        if not (0 <= s < S and -1 <= left < k and right < k):
            continue
        p = last[s] if left < 0 else kps[s, left]
        if right >= 0 and den > 0:
            p = _interp(p, kps[s, right], num, den)
        w, h = int(slots[s, 0]), int(slots[s, 1])
        if w > 0 and h > 0:
            out[r] = _normalise(p, w, h)
    new = last.copy()
    for s in range(S):
        if 0 <= slots[s, 2] < k:
            new[s] = kps[s, slots[s, 2]]
    return out, new
