"""CPU: the host side of moving slots between sessions -- DetectionBook / FrameBook slot transfer
against an uninterrupted book, the validation export_slots / import_slots apply before any device
work, StreamSlots serialisation, the header's C layout and the C-ABI error paths of
vp3d_stream_export / vp3d_stream_import."""
import io
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import videopose3d_b200 as vp
from videopose3d_b200 import _capi
from videopose3d_b200.streaming import (DetectionBook, FrameBook, StreamingSession, StreamSlots,
                                        weights_fingerprint)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _valid(out):
    return [int(v) for v in out if v >= 0]


@pytest.mark.parametrize("max_gap", [None, 0, 3, 20])
@pytest.mark.parametrize("seed", range(6))
def test_detection_book_moved_camera_matches_uninterrupted(max_gap, seed):
    """A camera runs in book U (S = 3, K = 2) with random detection masks, starts and ends; at a
    random call its slot is exported and imported into a running book B (S = 5, K = 3), where it
    goes on with the same inputs next to other random cameras.  Its releases, frame numbers, held
    counts and provisional frames are those of U's slot from then on."""
    rng = np.random.RandomState(seed)
    la = int(rng.choice([0, 4, 13]))
    U = DetectionBook(3, 2, max_gap, la)
    B = DetectionBook(5, 3, max_gap, la)
    src, dst = int(rng.randint(3)), int(rng.randint(5))
    move = int(rng.randint(0, 40))
    prov = max_gap is not None
    res = [(640, 480)] * 5
    started_b = np.zeros(5, bool)
    for call in range(80):
        k = int(rng.randint(1, 3))
        det_u = rng.rand(3, k) < rng.choice([0.2, 0.6, 0.95])
        start_u = [call == 0 or rng.rand() < 0.03 for _ in range(3)]
        end_u = [int(rng.randint(0, k + 1)) if rng.rand() < 0.04 and not start_u[s] else -1
                 for s in range(3)]
        if call >= 70:   # the camera's last video stays open into finish()
            start_u[src], end_u[src] = call == 70, -1
        if call == move:
            # B has been running; the camera replaces what slot dst held
            B.import_slots(U.export_slots([src]), [dst])
        det_b = rng.rand(5, k) < 0.7
        start_b = [not started_b[s] or rng.rand() < 0.03 for s in range(5)]
        end_b = [int(rng.randint(0, k + 1)) if rng.rand() < 0.04 and not start_b[s] else -1
                 for s in range(5)]
        started_b[:] = True
        if call >= move:
            det_b[dst] = det_u[src]
            start_b[dst], end_b[dst] = start_u[src], end_u[src]
        cu = U.push(det_u, start_u, end_u, res[:3], provisional=prov)
        cb = B.push(det_b, start_b, end_b, res, provisional=prov)
        if call < move:
            continue
        assert cu.frames[src] == cb.frames[dst], call
        assert cu.held[src] == cb.held[dst], call
        # (a draining tail advances with every push of its book, and the books make different
        # pushes: its frames come out at other calls, so they are compared while the video is open)
        if U.open[src]:
            assert _valid(cu.out[src]) == _valid(cb.out[dst]), call
            if prov:
                assert np.array_equal(cu.prov_frames[src], cb.prov_frames[dst]), call
    was_open = bool(U.open[src])
    fu, fb = U.finish(), B.finish()
    assert fu.frames[src] == fb.frames[dst]
    if was_open:
        assert _valid(fu.out[src]) == _valid(fb.out[dst])


@pytest.mark.parametrize("seed", range(8))
def test_frame_book_moved_slot_matches_uninterrupted(seed):
    """The same for FrameBook under push's start / end / count: a slot moved at any point (also
    while idle or draining) numbers its frames and provisional rows as the slot it left."""
    rng = np.random.RandomState(seed)
    la = int(rng.choice([0, 3, 121]))
    U, B = FrameBook(3, la), FrameBook(5, la)
    src, dst = int(rng.randint(3)), int(rng.randint(5))
    move = int(rng.randint(0, 60))
    for i in range(120):
        k = int(rng.randint(1, 3))
        su = rng.rand(3) < 0.05
        eu = np.where(rng.rand(3) < 0.05, rng.randint(0, k + 1, 3), -1)
        su &= eu != 0
        cu = rng.randint(0, k + 1, 3)
        sb = rng.rand(5) < 0.05
        eb = np.where(rng.rand(5) < 0.05, rng.randint(0, k + 1, 5), -1)
        cb = rng.randint(0, k + 1, 5)
        if i == move:
            B.import_slots(U.export_slots([src]), [dst])
        if i >= move:
            sb[dst], eb[dst], cb[dst] = su[src], eu[src], cu[src]
        fu, pu = U.push(k, su, eu, cu, provisional=True)
        fb, pb = B.push(k, sb, eb, cb, provisional=True)
        if i >= move:
            assert np.array_equal(fu[src], fb[dst]) and np.array_equal(pu[src], pb[dst]), i
    assert np.array_equal(U.finish()[src], B.finish()[dst])


def test_book_import_refuses_other_settings():
    a, b = DetectionBook(2, 2, 3, 4), DetectionBook(2, 2, 4, 4)
    with pytest.raises(ValueError, match="max_gap"):
        b.import_slots(a.export_slots([0]), [1])
    with pytest.raises(ValueError, match="lookahead"):
        DetectionBook(2, 2, 3, 5).import_slots(a.export_slots([0]), [1])
    with pytest.raises(ValueError, match="lookahead"):
        FrameBook(2, 1).import_slots(FrameBook(2, 0).export_slots([0]), [0])


def _bare_session(S=3, K=4, seed=0, augment=False):
    """The host-side attributes of a session, without the device state a real one allocates."""
    sess = StreamingSession.__new__(StreamingSession)
    torch.manual_seed(seed)
    sess.model = vp.TemporalModel(17, 2, 17, [3, 3], channels=64).eval()
    sess.streams, sess.max_frames, sess.lookahead = S, K, 4
    sess.device = torch.device("cuda", 0)
    sess.precision, sess.int8, sess.detections, sess.max_gap = "fp16", False, False, None
    sess.augment = augment
    sess._kps_src, sess._joints_src = vp.streaming.augment_maps(
        sess.model, augment, *(([4, 5, 6], [1, 2, 3]) * 2 if augment else ()))
    sess._versions = None
    return sess


def _slots_of(sess, n, device="cpu"):
    header = _capi.StreamSlotsHeader()
    header.n = n
    raw = torch.frombuffer(bytearray(bytes(header)), dtype=torch.uint8)
    return StreamSlots(torch.zeros(16 * n, dtype=torch.uint8, device=device), raw, sess._compat())


def test_slot_lists_are_checked_before_device_work():
    sess = _bare_session()
    assert sess._slot_list(range(3), True) == [0, 1, 2]
    assert sess._slot_list([2, 2], False) == [2, 2]
    assert sess._slot_list(torch.tensor([1, 0]), True) == [1, 0]
    with pytest.raises(ValueError, match="out of range"):
        sess._slot_list([0, 3], False)
    with pytest.raises(ValueError, match="out of range"):
        sess._slot_list([-1], False)
    with pytest.raises(ValueError, match="listed twice"):
        sess._slot_list([1, 0, 1], True)
    with pytest.raises(ValueError, match="no slots"):
        sess._slot_list([], False)
    with pytest.raises(TypeError, match="ints"):
        sess._slot_list([0.5], False)
    with pytest.raises(TypeError, match="ints"):
        sess._slot_list([True], False)


def test_import_validation_before_device_work():
    sess = _bare_session()
    state = _slots_of(sess, 2)
    with pytest.raises(TypeError, match="StreamSlots"):
        sess.import_slots(object(), [0, 1])
    with pytest.raises(ValueError, match="listed twice"):
        sess.import_slots(state, [1, 1])
    with pytest.raises(ValueError, match="out of range"):
        sess.import_slots(state, [0, 3])
    with pytest.raises(ValueError, match="2 exported"):
        sess.import_slots(state, [0])
    with pytest.raises(RuntimeError, match=r"\.to\("):
        sess.import_slots(state, [0, 1])   # the blob is on the CPU, the session on cuda:0
    # compatibility, on a session of the blob's device
    sess.device = torch.device("cpu")
    other = _bare_session()
    with torch.no_grad():
        other.model.layers_conv[1].weight[0, 0, 0] += 1e-3   # one perturbed parameter
    with pytest.raises(ValueError, match="weights differs"):
        sess.import_slots(_slots_of(other, 2), [0, 1])
    for attr, value, key in (("augment", True, "augment"), ("max_gap", 3, "max_gap"),
                             ("precision", "bf16", "precision"), ("lookahead", 0, "lookahead"),
                             ("detections", True, "detections")):
        o = _bare_session()
        setattr(o, attr, value)
        with pytest.raises(ValueError, match=f"{key} differs"):
            sess.import_slots(_slots_of(o, 2), [0, 1])
    aug, aug2 = _bare_session(augment=True), _bare_session(augment=True)
    aug2._kps_src = aug2._kps_src[::-1].copy()
    aug.device = torch.device("cpu")
    with pytest.raises(ValueError, match="kps_src differs"):
        aug.import_slots(_slots_of(aug2, 1), [0])
    wide = _bare_session()
    wide.model = vp.TemporalModel(17, 2, 17, [3, 3, 3], channels=64).eval()
    with pytest.raises(ValueError, match="architecture differs"):
        sess.import_slots(_slots_of(wide, 2), [0, 1])


def test_weights_fingerprint_follows_values_not_objects():
    a, b = _bare_session(seed=1).model, _bare_session(seed=2).model
    assert weights_fingerprint(a) != weights_fingerprint(b)
    b.load_state_dict(a.state_dict())
    assert weights_fingerprint(a) == weights_fingerprint(b)
    before = weights_fingerprint(a)
    with torch.no_grad():
        a.layers_bn[0].running_var[3] *= 2
    assert weights_fingerprint(a) != before


def test_stream_slots_survive_save_and_load():
    sess = _bare_session()
    state = _slots_of(sess, 3)
    state.blob[:] = torch.arange(48, dtype=torch.uint8)
    state.book = DetectionBook(4, 2, 3, 4).export_slots([1, 2, 3])
    buf = io.BytesIO()
    torch.save(state, buf)
    buf.seek(0)
    back = torch.load(buf)   # weights_only (torch's default)
    assert isinstance(back, StreamSlots) and len(back) == 3
    assert torch.equal(back.blob, state.blob) and torch.equal(back.header, state.header)
    assert back.compat == state.compat
    assert back.book["max_gap"] == 3 and torch.equal(back.book["seen"], state.book["seen"])
    assert back.to("cpu").blob.device.type == "cpu"


def test_slots_header_matches_the_c_layout(tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    cls = _capi.StreamSlotsHeader
    name = "vp3d_stream_slots_header"
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "vp3d_b200.h"', 'int main(void) {',
             f'  printf("size %zu\\n", sizeof({name}));']
    for f, _ in cls._fields_:
        lines.append(f'  printf("{f} %zu\\n", offsetof({name}, {f}));')
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                           str(exe)])
    out = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(out["size"]) == _capi.ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(out[f]) == getattr(cls, f).offset, f


@pytest.mark.parametrize("entry", ["vp3d_stream_export", "vp3d_stream_import"])
def test_transfer_entries_report_errors_without_gpu(entry):
    """Argument checks of vp3d_stream_export / _import run before any device work, under their own
    names."""
    lib = _capi.load()
    fn = getattr(lib, entry)
    what = entry[len("vp3d_"):].encode()
    fake = 1 << 20   # never dereferenced: the checks fail first
    slots = np.zeros(2, np.int32)
    sp = slots.ctypes.data
    header = _capi.StreamSlotsHeader()
    hp = _capi.ctypes.byref(header)
    cases = [((fake, None, sp, 2, fake, 1 << 20, hp), b"null state"),
             ((None, fake, sp, 2, fake, 1 << 20, hp), b"null plan"),
             ((fake, fake, sp, 0, fake, 1 << 20, hp), b"n must be >= 1"),
             ((fake, fake, None, 2, fake, 1 << 20, hp), b"null slots, blob or header"),
             ((fake, fake, sp, 2, None, 1 << 20, hp), b"null slots, blob or header"),
             ((fake, fake, sp, 2, fake, 1 << 20, None), b"null slots, blob or header"),
             ((fake, fake, sp, 2, fake + 8, 1 << 20, hp), b"16-byte aligned")]
    for args, msg in cases:
        assert fn(*args, None) == -1, msg
        err = lib.vp3d_last_error()
        assert what + b": " in err and msg in err, err
    assert lib.vp3d_stream_slot_bytes(None, 0) == 0
