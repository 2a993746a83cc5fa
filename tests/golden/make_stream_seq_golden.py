"""Golden outputs for streaming several sequences of different lengths through one session
(StreamingSession.predict, or push with `end`), produced by the REAL reference.

    python tests/golden/make_stream_seq_golden.py [--reference DIR]

Writes `tests/golden/stream_seq/*.npz`.  Each case is run.py's evaluation loop (run.py:186-193,
652-683) over a list of sequences: the reference's `common/generators.py` UnchunkedGenerator over
all of them, the reference's `common/model.py` TemporalModel (eval) on every batch it yields, and
with test-time augmentation the mirror undone on the second output and the two averaged
(run.py:674-680; the trajectory model only negates x, :678).  Joint lists: the 17-joint Human3.6M
ones.  The lengths include a single frame and sequences shorter than the receptive field.  Entries:
  x        (sum T, J, F) float32   the 2-D input sequences, concatenated
  y        (sum T, J_out, 3) float32   the reference's predictions, concatenated
  lengths  (n,) int64   frames of every sequence
  meta     json: fw, causal, dense, C, J, F, Jout, augment, lengths, seed
`make_case(name, reference_dir)` regenerates one case (used by the CPU test that checks the files).
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "stream_seq")

# Human3.6M's 17-joint skeleton (the reference's kps_left/right and joints_left/right, run.py:67-69)
LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]

# name -> (filter widths, causal, dense, channels, J_out, augment, lengths, seed); RF 27, 45, 63
# (3,3,7: run.py's documented example) and 9 (3,1,3: a 1-tap block, whose ring keeps no history)
CASES = {
    "seq_333_c64_tta": ([3, 3, 3], False, False, 64, 17, True, [40, 1, 13, 29, 5, 2], 61),
    "seq_333_c64_causal": ([3, 3, 3], True, False, 64, 17, False, [33, 7, 1, 26, 50], 62),
    "seq_353_c128_traj_tta": ([3, 5, 3], False, False, 128, 1, True, [1, 60, 44, 3, 17], 63),
    "seq_337_c64_tta": ([3, 3, 7], False, False, 64, 17, True, [70, 1, 20, 63, 2, 64], 64),
    "seq_313_c64_causal": ([3, 1, 3], True, False, 64, 17, False, [15, 1, 9, 30, 4, 8], 65),
}


def make_case(name, reference_dir):
    import torch
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    if reference_dir not in sys.path:
        sys.path.insert(0, reference_dir)
    from common.generators import UnchunkedGenerator
    from common.model import TemporalModel
    from oracle import temporal_model_oracle as orc
    fw, causal, dense, C, jout, augment, lengths, seed = CASES[name]
    J, F = 17, 2
    use_trajectory_model = jout == 1
    kps_left, kps_right = list(LEFT), list(RIGHT)
    joints_left, joints_right = list(LEFT), list(RIGHT)
    torch.set_num_threads(1)
    model = TemporalModel(J, F, jout, filter_widths=fw, causal=causal, dropout=0.25, channels=C,
                          dense=dense)
    model.load_state_dict(orc.make_state_dict(J, F, jout, fw, C, dense=dense, seed=seed))
    xs = [orc.make_input(1, T, J, F, seed=seed + 1 + i)[0].numpy() for i, T in enumerate(lengths)]
    # run.py:186-193: receptive field -> pad, causal shift
    receptive_field = model.receptive_field()
    pad = (receptive_field - 1) // 2
    causal_shift = pad if causal else 0
    gen = UnchunkedGenerator(None, None, xs, pad=pad, causal_shift=causal_shift, augment=augment,
                             kps_left=kps_left, kps_right=kps_right, joints_left=joints_left,
                             joints_right=joints_right)
    ys = []
    with torch.no_grad():   # run.py:657-683, every batch (one per sequence)
        model.eval()
        for _, batch, batch_2d in gen.next_epoch():
            inputs_2d = torch.from_numpy(batch_2d.astype('float32'))
            predicted_3d_pos = model(inputs_2d)
            if gen.augment_enabled():
                predicted_3d_pos[1, :, :, 0] *= -1
                if not use_trajectory_model:
                    predicted_3d_pos[1, :, joints_left + joints_right] = \
                        predicted_3d_pos[1, :, joints_right + joints_left]
                predicted_3d_pos = torch.mean(predicted_3d_pos, dim=0, keepdim=True)
            ys.append(predicted_3d_pos.squeeze(0).cpu().numpy())
    assert [len(y) for y in ys] == lengths
    meta = dict(fw=fw, causal=causal, dense=dense, C=C, J=J, F=F, Jout=jout, augment=augment,
                lengths=lengths, seed=seed)
    return {"x": np.concatenate(xs).astype(np.float32), "y": np.concatenate(ys).astype(np.float32),
            "lengths": np.array(lengths, np.int64), "meta": np.array(json.dumps(meta))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=None)
    args = ap.parse_args()
    ref = args.reference
    if ref is None:
        sys.path.insert(0, ROOT)
        from oracle import stage_ref
        ref = stage_ref.reference_dir()
    if ref is None:
        raise SystemExit("no reference checkout: pass --reference")
    os.makedirs(OUT, exist_ok=True)
    for name in CASES:
        case = make_case(name, ref)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **case)
        print(f"{path}: y {case['y'].shape}, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
