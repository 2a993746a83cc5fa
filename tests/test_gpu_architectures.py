"""GPU: every model path on architectures beyond filter widths 3 and 5, layer by layer against
float64, with the gates of the per-path modules.

The widths enter the tap-major row permutation, the strided trim and residual regions, the expand's
K padding (J F w0 -> a multiple of 64), the dilated taps and their transposed data gradients, the
stream rings' histories (w0 - 1 and 2 pad_i: none for a width-1 layer), the clip chain's RF - 1
padding rows and mixed's per-layer split.  The table:

    a337   3,3,7 at C = 1024     run.py's documented example (RF 63): a width-7 block at
                                 dilation 9 (pad 27), 128-wide tiles
    a355c  3,5,5 causal, C = 100 the other documented example: causal shifts 6 and 30, padded
                                 channels
    a733   7,3,3 at C = 256      expand width 7: strided K0 = 238 -> 256, 7 dilated expand taps,
                                 the input gradient's strided tail
    a313   3,1,3 at C = 128      a 1-tap block: pad 0, the whole input as residual, a ring with no
                                 history
    a133   1,3,3 at C = 128      expand width 1: K0 = 34 -> 64, ring 0 with no history
    j32    3,3,3, J = 32, F = 3  the full Human3.6M skeleton in 3-D: K0 = 288 -> 320 (five
                                 k-blocks), shrink of 96 -> 128 columns
    d337   3,3,7 dense, C = 128  7- and 55-tap blocks

and the paths:
1. eval, layer by layer (test_gpu_eval_layers.test_eval_layers: per-GEMM float64 bounds, the
   replay's bit tie and launch count, the layout against forward_numpy) in fp16, bf16, bf16x3 and
   mixed, on the cone (T = RF), the dilated (T > RF, ragged last tile) and the strided schedule;
   the gate is shown to reject a width-7 block's taps read in reverse order and a dilated launch's
   taps one frame off;
2. int8 (test_gpu_eval_layers_int8) with every block in int8, and a set_int8_blocks mask with an
   fp16 block before an int8 one (test_gpu_int8_blocks.test_layers); the int32 overflow guard at
   its boundary: dense 3,3,3,3,3 (a 163-tap block) at C = 406 runs and passes the int8 gates,
   C = 407 is refused, and one 163-tap u8 x s8 launch whose largest sum is 2 143 174 530
   (0.2 % below 2^31) equals the exact sum's epilogue bit for bit;
3. training, layer by layer (test_gpu_train_layers.test_train_layers) in bf16 and bf16x3, dropout
   0 and 0.25, with dx and with frozen-BatchNorm dx; TemporalModel dilated training of a337 with
   two or three 128-row tiles per sample, the last one ragged (run.py's --stride 200), and the
   dense d337;
4. streaming sessions equal to the offline forward bit for bit, plain and with flip augmentation,
   k in {1, 7}, slots starting mid-stream, `end` on live slots and finish(); the check is shown to
   reject a sequence whose first frame is missing from the history;
5. predict(clips) equal to each clip's own forward bit for bit, with 1-, 2- and RF-frame clips;
6. the optimizer's fused re-pack equal to the plain update and vp3d_set_weights (a733, j32).
"""
import ctypes

import numpy as np
import pytest
import torch

import eval_replay as er
from oracle import temporal_model_oracle as orc
import test_gpu_adam_step as tas
import test_gpu_eval_layers as tel
import test_gpu_eval_layers_int8 as tei
from test_gpu_int8 import _launch
import test_gpu_int8_blocks as tib
import test_gpu_predict as tp
import test_gpu_streaming_seq as tss
import test_gpu_train_layers as ttl
import videopose3d_b200 as vp
from videopose3d_b200 import _capi

pytestmark = pytest.mark.gpu

TM, OPT = "TemporalModel", "TemporalModelOptimized1f"


def _cfg(cls, fw, C, J=17, F=2, Jout=17, causal=False, dense=False):
    return dict(cls=cls, fw=list(fw), C=C, J=J, F=F, Jout=Jout, causal=causal, dense=dense)


# arc id -> (filter widths, model keywords)
ARCHS = {
    "a337": ([3, 3, 7], dict(C=1024)),
    "a355c": ([3, 5, 5], dict(C=100, causal=True)),
    "a733": ([7, 3, 3], dict(C=256)),
    "a313": ([3, 1, 3], dict(C=128)),
    "a133": ([1, 3, 3], dict(C=128)),
    "j32": ([3, 3, 3], dict(C=256, J=32, F=3, Jout=32)),
    "d337": ([3, 3, 7], dict(C=128, dense=True)),
}


def _arch(arc, cls=TM):
    fw, kw = ARCHS[arc]
    return _cfg(cls, fw, **kw)


def _rf(arc):
    return orc.arch(ARCHS[arc][0])["receptive_field"]


# ------------------------------------------------------------------------------------ 1. eval
# (id, cfg, N, T): cone (T = RF), dilated (T > RF: 128-row tiles per sample, the last one ragged),
# strided (TemporalModelOptimized1f; a733 also with a strided tail T = 68 = 7 * 9 + 5)
EVAL = [
    ("a337_cone", _arch("a337"), 64, 63),
    ("a337_dilated", _arch("a337"), 4, 262),
    ("a337_opt", _arch("a337", OPT), 64, 63),
    ("a355c_cone", _arch("a355c"), 100, 75),
    ("a355c_dilated", _arch("a355c"), 8, 200),
    ("a355c_opt", _arch("a355c", OPT), 100, 75),
    ("a733_cone", _arch("a733"), 100, 63),
    ("a733_dilated", _arch("a733"), 6, 190),
    ("a733_opt_t68", _arch("a733", OPT), 100, 68),
    ("a313_cone", _arch("a313"), 300, 9),
    ("a313_dilated", _arch("a313"), 8, 150),
    ("a313_opt", _arch("a313", OPT), 300, 9),
    ("a133_cone", _arch("a133"), 300, 9),
    ("a133_dilated", _arch("a133"), 8, 150),
    ("a133_opt", _arch("a133", OPT), 300, 9),
    ("j32_cone", _arch("j32"), 200, 27),
    ("j32_dilated", _arch("j32"), 8, 150),
    ("j32_opt", _arch("j32", OPT), 200, 27),
    ("d337_dense", _arch("d337"), 4, 150),
]
EVAL_PARAMS = [pytest.param(*c, p, id=f"{c[0]}-{p}") for c in EVAL for p in er.PRECISIONS]


def _rejects(lc, plan, case):
    """True when test_gpu_eval_layers' per-launch gate fails for `lc`."""
    try:
        tel._check_launch(lc, plan, case)
    except AssertionError:
        return True
    return False


def _wrong(lc, w=None, **desc):
    return er.Launch(lc.name, dict(lc.desc, **desc), lc.a, lc.w if w is None else w, lc.scale,
                     lc.shift, res=lc.res, out=lc.out, out_f32=lc.out_f32)


@pytest.mark.parametrize("case,cfg,N,T,precision", EVAL_PARAMS)
def test_eval_layers(cuda_device, case, cfg, N, T, precision):
    tel.test_eval_layers(cuda_device, case, cfg, N, T, precision)
    # the gate rejects plausible wrong answers on the same launches
    sd = tel._state_dict(tel._key(cfg))
    x = orc.make_input(N, T, cfg["J"], cfg["F"], seed=1).to(cuda_device)
    with torch.no_grad():
        rep = er.replay(sd, cfg, x, precision, er.gpu_gemm)
    seven = [lc for lc in rep.launches if lc.desc["taps"] == 7]
    for lc in seven[:1]:   # a width-7 conv with its taps read in reverse order
        assert _rejects(_wrong(lc, w=lc.w.flip(1)), rep.plan, case), \
            f"{case}: {lc.name} passes with its taps reversed"
    dil = [lc for lc in rep.launches
           if lc.desc["per_sample_tiles"] and lc.desc["taps"] > 1 and lc.desc["tap_row_step"] > 0]
    for lc in dil[-1:]:    # a dilated conv whose taps are one frame closer together
        d = lc.desc["tap_row_step"]
        assert _rejects(_wrong(lc, tap_row_step=d - 1), rep.plan, case), \
            f"{case}: {lc.name} passes with dilation {d - 1} for {d}"
    # (the strided expand merges its taps into one K: 7,3,3 has a 7-tap launch when dilated only)
    if 7 in cfg["fw"][1:] or (cfg["fw"][0] == 7 and not rep.plan.strided):
        assert seven, f"{case}: no 7-tap launch"
    if not rep.plan.strided:
        assert dil, f"{case}: no dilated launch"


# ------------------------------------------------------------------------------------ 2. int8
INT8 = [
    ("a337_dilated", _arch("a337"), 4, 262),
    ("a337_opt", _arch("a337", OPT), 64, 63),
    ("a355c_dilated", _arch("a355c"), 8, 200),
    ("a733_dilated", _arch("a733"), 6, 190),
    ("a733_opt_t68", _arch("a733", OPT), 100, 68),
    ("a313_dilated", _arch("a313"), 8, 150),
    ("a313_opt", _arch("a313", OPT), 300, 9),
    ("a133_dilated", _arch("a133"), 8, 150),
    ("a133_opt", _arch("a133", OPT), 300, 9),
    ("j32_cone", _arch("j32"), 200, 27),
    ("j32_dilated", _arch("j32"), 8, 150),
    ("d337_dense", _arch("d337"), 4, 150),
    # the int32 guard's largest accepted channel count for a 163-tap block (2 143 174 530 < 2^31)
    ("dense_33333_c406", _cfg(TM, [3, 3, 3, 3, 3], 406, dense=True), 1, 260),
]


@pytest.mark.parametrize("case,cfg,N,T", INT8, ids=[c[0] for c in INT8])
def test_eval_layers_int8(cuda_device, case, cfg, N, T):
    tei.test_eval_layers_int8(cuda_device, case, cfg, N, T, None)


# block 1 in fp16, block 2 in int8: the quantise pass between them
MASKED = [(c[0], c[1], c[2], c[3]) for c in INT8
          if c[0] in ("a337_dilated", "a733_opt_t68", "a313_dilated", "a133_opt")]


@pytest.mark.parametrize("case,cfg,N,T", MASKED, ids=[c[0] for c in MASKED])
def test_int8_fp16_block_before_int8_block(cuda_device, case, cfg, N, T):
    tib.test_layers(cuda_device, case, cfg, N, T, [2])


def _dense_33333(C):
    return vp.TemporalModel(17, 2, 17, [3, 3, 3, 3, 3], dense=True, dropout=0.0, channels=C)


def test_int8_overflow_guard_boundary(cuda_device):
    """163 x 406 x 255 x 127 = 2 143 174 530 < 2^31 <= 163 x 407 x 255 x 127 = 2 148 453 285."""
    assert 163 * 406 * 255 * 127 == 2143174530 < 2 ** 31 <= 163 * 407 * 255 * 127
    lib = _capi.load()
    for C, want in ((406, 0), (407, -2)):   # VP3D_ERR_UNSUPPORTED
        cfg = _dense_33333(C)._config("int8")
        handle = ctypes.c_void_p()
        with torch.cuda.device(cuda_device):
            st = lib.vp3d_plan_create(ctypes.byref(cfg), ctypes.byref(handle))
        assert st == want, (C, st, lib.vp3d_last_error())
        if st == 0:
            lib.vp3d_plan_destroy(handle)
        else:
            assert b"overflow" in lib.vp3d_last_error()
    m = _dense_33333(407).to(cuda_device).eval()
    m.set_precision("int8").load_int8_calibration(torch.ones(8))
    with pytest.raises(NotImplementedError, match="overflow"):
        with torch.no_grad():
            m(orc.make_input(1, 243, seed=1).to(cuda_device))


def test_int8_gemm_at_the_int32_bound(cuda_device):
    """One u8 x s8 launch of 163 taps x 406 live channels (k_per_tap 512), A all 255 and W 127 on
    most output columns: the largest int32 sum is 2 143 174 530.  Each output is fmaf(fp32(acc),
    scale', shift) on the exact integer sum, ReLU, then fp16, bit for bit; a wrap-around anywhere
    in the accumulation flips the sign and ReLU makes it 0."""
    dev = cuda_device
    taps, c_live, a_ld, k_pad, n_pad, out_rows = 163, 406, 448, 512, 64, 256
    a_rows = out_rows + taps - 1
    a = torch.zeros(a_rows, a_ld, dtype=torch.uint8)
    a[:, :c_live] = 255
    wcol = torch.full((n_pad,), 127, dtype=torch.int64)
    wcol[[3, 17, 40, 63]] = torch.tensor([126, 1, 64, 100])   # a few smaller, distinct sums
    w = torch.zeros(taps, n_pad, k_pad, dtype=torch.int8)
    w[:, :, :c_live] = wcol.to(torch.int8)[None, :, None]
    acc = taps * c_live * 255 * wcol                          # exact, int64
    assert int(acc.max()) == 2143174530
    scale = torch.full((n_pad,), 2.0 ** -16)                  # 2^31 * 2^-16 = 32768 < 65504
    shift = torch.linspace(-0.5, 0.5, n_pad)
    res = torch.zeros(out_rows, n_pad, dtype=torch.float16, device=dev)
    out = torch.full((out_rows, n_pad), float("nan"), dtype=torch.float16, device=dev)
    _launch(a.to(dev), 1, a_rows, a_ld, w.to(dev), taps, k_pad, n_pad, per_sample=False,
            tap_row_step=1, out_rows=out_rows, precision=_capi.VP3D_PRECISION_INT8,
            scale=scale.to(dev), shift=shift.to(dev), res=res, out=out)
    v = er.fma_f32(torch.from_numpy(acc.numpy().astype(np.float32)), scale, shift).clamp_min(0)
    exp = v.half()[None].expand(out_rows, n_pad)
    got = out.cpu()
    n = int((got.view(torch.int16) != exp.view(torch.int16)).sum())
    assert n == 0, f"{n} of {got.numel()} outputs differ from the exact sum's epilogue: " \
        f"row 0 got {got[0].tolist()}, want {exp[0].tolist()}"
    assert float(got.min()) > 0


# -------------------------------------------------------------------------------- 3. training
# (id, cfg, N, T, options)
TRAIN = [
    ("a337_opt", _arch("a337", OPT), 16, 63, {}),
    ("a355c_opt", _arch("a355c", OPT), 100, 75, {}),
    ("a733_opt", _arch("a733", OPT), 64, 63, {}),
    ("a733_opt_dx_t68", _arch("a733", OPT), 64, 68, dict(dx=True)),
    ("a313_opt", _arch("a313", OPT), 300, 9, {}),
    ("a313_opt_frozen_dx", _arch("a313", OPT), 300, 9, dict(dx=True, frozen=True)),
    ("a133_opt_dx", _arch("a133", OPT), 300, 9, dict(dx=True)),
    ("j32_opt", _arch("j32", OPT), 200, 27, {}),
    ("j32_opt_frozen_dx", _arch("j32", OPT), 200, 27, dict(dx=True, frozen=True)),
    # run.py --stride 200: 200 output frames per sample, 200 to 260 rows per layer: two or three
    # 128-row tiles per sample, the last one ragged
    ("a337_dilated_stride200", _arch("a337"), 4, 62 + 200, {}),
    ("a337_dilated_frozen_dx", _arch("a337"), 2, 62 + 200, dict(dx=True, frozen=True)),
    ("d337_dense", _arch("d337"), 4, 100, {}),
    ("d337_dense_dx", _arch("d337"), 4, 100, dict(dx=True)),
]
TRAIN_PARAMS = [pytest.param(*c, prec, p, id=f"{c[0]}-{prec}-p{p}")
                for c in TRAIN for prec in ("bf16", "bf16x3")
                for p in ((0.0,) if c[4].get("frozen") else (0.0, ttl.P))]


@pytest.mark.parametrize("case,cfg,N,T,opt,precision,p", TRAIN_PARAMS)
def test_train_layers(cuda_device, case, cfg, N, T, opt, precision, p):
    ttl.test_train_layers(cuda_device, case, cfg, N, T, opt, precision, p)


# ------------------------------------------------------------------------------- 4. streaming
def _model(dev, arc, precision, seed):
    fw, kw = ARCHS[arc]
    cfg = _cfg(TM, fw, **kw)
    m = vp.TemporalModel(cfg["J"], cfg["F"], cfg["Jout"], filter_widths=fw, causal=cfg["causal"],
                         dropout=0.0, channels=cfg["C"], dense=cfg["dense"])
    m.load_state_dict(orc.make_state_dict(cfg["J"], cfg["F"], cfg["Jout"], fw, cfg["C"],
                                          dense=cfg["dense"], seed=seed))
    return m.to(dev).eval().set_precision(precision)


def _first_frame_missing_is_rejected(m, out, augment):
    """The bit-for-bit check fails for a sequence whose first frame is missing from the history
    (the edge padding taken from frame 1): what a ring one frame short gives at a start."""
    for x, rows, dropped in out.values():
        if dropped or len(x) < 3 or len(rows) != len(x):
            continue
        got = torch.stack([rows[f] for f in range(len(x))])
        assert not torch.equal(got[1:], tss._offline(m, x[1:], augment))
        return
    raise AssertionError("no complete sequence of 3 frames or more")


@pytest.mark.parametrize("arc", list(ARCHS))
def test_streaming(cuda_device, arc):
    m = _model(cuda_device, arc, "fp16", seed=31)
    hist = vp.streaming.ring_history(ARCHS[arc][0], dense=ARCHS[arc][1].get("dense", False))
    if arc in ("a313", "a133"):
        assert 0 in list(hist), hist
    rng = np.random.RandomState(len(arc))
    rf = _rf(arc)
    S = 4
    for K in (1, 7):
        seqs = {s: [int(v) for v in rng.randint(2, rf + 20, 2)] for s in range(S)}
        out = tss._live_session(m, S, K, seqs, seed=K + 40)
        tss._check_live(m, out)
        if K == 7:
            _first_frame_missing_is_rejected(m, out, False)
    # flip augmentation in bf16x3, and finish() with slots ended, open and idle
    m.set_precision("bf16x3")
    seqs = {s: [int(v) for v in rng.randint(2, rf + 20, 3)] for s in range(S)}
    tss._check_live(m, tss._live_session(m, S, 7, seqs, seed=50, augment=True), augment=True)
    out = tss._live_session(m, S, 7, seqs, seed=51, augment=True, finish_at=12)
    tss._check_live(m, out, augment=True, complete=False)


# ---------------------------------------------------------------------------------- 5. clips
@pytest.mark.parametrize("augment", [False, True])
@pytest.mark.parametrize("arc", list(ARCHS))
def test_predict_clips(cuda_device, arc, augment):
    m = _model(cuda_device, arc, "fp16", seed=33)
    J, F = m.num_joints_in, m.in_features
    rf = _rf(arc)
    rng = np.random.RandomState(34)
    lengths = [1, 2, rf, rf + 1] + [int(v) for v in rng.randint(1, 3 * rf, 8)]
    clips = [orc.make_input(1, T, J, F, seed=350 + i)[0].to(cuda_device)
             for i, T in enumerate(lengths)]
    ys = tp._predict(m, clips, augment)
    assert m.last_predict_launches == 2 * (len(ARCHS[arc][0]) - 1) + 4   # one chain
    for x, y in zip(clips, ys):
        assert tuple(y.shape) == (len(x), m.num_joints_out, 3)
        if len(x) >= 2:
            assert torch.equal(y, tp._offline(m, x, augment)), len(x)
    # every clip, 1-frame ones included: a streaming session computes the same bits
    sess = m.streaming(streams=3, max_frames=7, augment=augment, **tp._lists(m, augment))
    for a, b in zip(ys, sess.predict(clips)):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------ 6. optimizer re-pack
REPACK = [("a733_opt", _arch("a733", OPT), 16, 63), ("j32_opt", _arch("j32", OPT), 40, 27)]


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("case,cfg,N,T", REPACK, ids=[c[0] for c in REPACK])
def test_fused_repack_matches_plain_update(cuda_device, case, cfg, N, T, precision):
    tas.test_fused_repack_matches_plain_update(cuda_device, case, cfg, N, T, precision, 0.25)
