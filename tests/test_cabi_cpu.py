"""CPU: the C-ABI library loads and exports every symbol include/vp3d_b200.h declares; the Python
module mirrors the reference's nn.Module contract (constructor, attributes, state_dict layout) and
refuses to compute without CUDA (no fallback)."""
import os
import re

import pytest
import torch

import videopose3d_b200 as vp
from videopose3d_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    text = open(os.path.join(ROOT, "include", "vp3d_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(vp3d_[a-z_0-9]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    if not os.path.exists(_capi.lib_path()):
        import __graft_entry__ as g
        g.build()
    lib = _capi.load()
    declared = _declared_functions()
    assert len(declared) >= 14
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
        assert name in _capi.SIGNATURES, f"{name} has no ctypes signature"
    assert lib.vp3d_version() == 200
    assert sorted(_capi.SIGNATURES) == declared


def test_struct_sizes_match_header_layout():
    # vp3d_config: 4 ints + int[8] + 5 ints
    assert _capi.ctypes.sizeof(_capi.Config) == 4 * (4 + 8 + 5)
    # vp3d_weights: 1 + 4 + 14 + 14*4 + 2 pointers
    assert _capi.ctypes.sizeof(_capi.Weights) == 8 * (1 + 4 + 14 + 56 + 2)


def test_ctypes_structs_match_the_c_header(tmp_path):
    """sizeof / offsetof of every struct the Python host passes by pointer, measured by compiling the
    public header with the C compiler, against the ctypes mirrors in _capi.py."""
    import shutil
    import subprocess
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    ct = _capi.ctypes
    pairs = {"vp3d_config": _capi.Config, "vp3d_weights": _capi.Weights, "vp3d_grads": _capi.Grads,
             "vp3d_conv_desc": _capi.ConvDesc, "vp3d_gather_desc": _capi.GatherDesc,
             "vp3d_adam_tensor": _capi.AdamTensor, "vp3d_wgrad_desc": _capi.WgradDesc}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "vp3d_b200.h"', 'int main(void) {']
    for cname, cls in pairs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    include = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    subprocess.check_call([cc, "-std=c99", "-I", include, str(src), "-o", str(exe)])
    out = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    for cname, cls in pairs.items():
        assert int(out[cname]) == ct.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert int(out[f"{cname}.{fname}"]) == getattr(cls, fname).offset, f"{cname}.{fname}"


def test_plan_create_reports_errors_without_gpu():
    lib = _capi.load()
    cfg = _capi.Config()
    cfg.num_joints_in, cfg.in_features, cfg.num_joints_out = 17, 2, 17
    cfg.num_widths = 2
    cfg.filter_widths[0], cfg.filter_widths[1] = 3, 4
    cfg.channels = 1024
    h = _capi.ctypes.c_void_p()
    st = lib.vp3d_plan_create(_capi.ctypes.byref(cfg), _capi.ctypes.byref(h))
    assert st == -1 and b"odd filter widths" in lib.vp3d_last_error()
    cfg.filter_widths[1] = 3
    cfg.channels = 0
    st = lib.vp3d_plan_create(_capi.ctypes.byref(cfg), _capi.ctypes.byref(h))
    assert st == -1 and b"channels must be positive" in lib.vp3d_last_error()
    cfg.channels = 100   # any positive channel count is accepted (padded to 64 internally)
    if not torch.cuda.is_available():
        st = lib.vp3d_plan_create(_capi.ctypes.byref(cfg), _capi.ctypes.byref(h))
        assert st == -3  # VP3D_ERR_CUDA: reported, not a crash and not a CPU fallback


def test_gather_entry_points_report_errors_without_gpu():
    """vp3d_gather_windows / vp3d_gather_cameras validate their arguments before any launch."""
    ct = _capi.ctypes
    lib = _capi.load()
    assert ct.sizeof(_capi.GatherDesc) == 6 * 8 + 5 * 4 + 4  # 6 pointers, 5 int32, tail padding
    assert lib.vp3d_gather_windows(None, None) == -1
    d = _capi.GatherDesc()
    d.n_windows, d.frames, d.joints, d.features = 1, 1, 100, 3  # 300 elements per frame > 256
    assert lib.vp3d_gather_windows(ct.byref(d), None) == -2
    d.joints = 17
    assert lib.vp3d_gather_windows(ct.byref(d), None) == -1   # null pointers
    assert b"null pointer" in lib.vp3d_last_error()
    d.n_windows = 0
    assert lib.vp3d_gather_windows(ct.byref(d), None) == 0    # empty batch: no-op, no launch
    assert lib.vp3d_gather_cameras(None, 9, None, 0, None, None) == 0
    assert lib.vp3d_gather_cameras(None, 9, None, 3, None, None) == -1


def test_step_op_entry_points_report_errors_without_gpu():
    ct = _capi.ctypes
    lib = _capi.load()
    assert ct.sizeof(_capi.AdamTensor) == 48
    assert lib.vp3d_adam_step(None, 0, 1, 1e-3, 0.9, 0.999, 1e-8, 0.0, None) == 0  # nothing to do
    assert lib.vp3d_adam_step(None, 2, 1, 1e-3, 0.9, 0.999, 1e-8, 0.0, None) == -1
    row = (_capi.AdamTensor * 1)()
    row[0].numel = 10
    assert lib.vp3d_adam_step(row, 1, 0, 1e-3, 0.9, 0.999, 1e-8, 0.0, None) == -1
    assert b"step must be >= 1" in lib.vp3d_last_error()
    assert lib.vp3d_adam_step(row, 1, 1, 1e-3, 1.0, 0.999, 1e-8, 0.0, None) == -1  # beta1 = 1
    assert lib.vp3d_adam_step(row, 1, 1, 1e-3, 0.9, 0.999, 1e-8, 0.0, None) == -1  # null pointers
    assert b"null pointer" in lib.vp3d_last_error()
    assert lib.vp3d_mpjpe_fwd_bwd(None, None, None, 4, 3, None, None, None) == -1
    assert lib.vp3d_mpjpe_fwd_bwd(None, None, None, 4, 0, None, None, None) == -1
    assert lib.vp3d_projected_mpjpe_fwd_bwd(None, None, None, None, 4, 1, 17, 0, None, None, None,
                                            None) == -1
    assert lib.vp3d_projected_mpjpe_fwd_bwd(None, None, None, None, 4, 0, 17, 0, None, None, None,
                                            None) == -1


def test_fused_adam_contract_without_gpu():
    """Same state_dict layout as torch.optim.Adam (checkpoints interchange, run.py:295-296, 600-608);
    CPU tensors are refused rather than routed through torch."""
    from videopose3d_b200.optim import FusedAdam
    ps = [torch.nn.Parameter(torch.randn(5, 3)), torch.nn.Parameter(torch.randn(7))]
    ref = torch.optim.Adam(ps, lr=2e-3, amsgrad=True)
    for p in ps:
        p.grad = torch.randn_like(p)
    ref.step()
    ours = FusedAdam(ps, lr=1e-3, amsgrad=True)
    ours.load_state_dict(ref.state_dict())
    assert ours.param_groups[0]["lr"] == 2e-3 and ours.param_groups[0]["amsgrad"] is True
    for p in ps:
        assert set(ours.state[p]) == {"step", "exp_avg", "exp_avg_sq", "max_exp_avg_sq"}
        assert float(ours.state[p]["step"]) == 1.0
    back = torch.optim.Adam(ps, lr=1e-3, amsgrad=True)
    back.load_state_dict(ours.state_dict())
    assert torch.equal(back.state[ps[0]]["exp_avg"], ref.state[ps[0]]["exp_avg"])
    with pytest.raises(RuntimeError, match="CUDA float32"):
        ours.step()
    with pytest.raises(ValueError):
        FusedAdam(ps, lr=-1.0)
    from videopose3d_b200 import loss as vloss
    with pytest.raises(RuntimeError, match="CUDA float32"):
        vloss.mpjpe(torch.zeros(2, 1, 17, 3), torch.zeros(2, 1, 17, 3))


@pytest.mark.parametrize("cls,kw", [
    (vp.TemporalModel, dict(filter_widths=[3, 3, 3], causal=False)),
    (vp.TemporalModel, dict(filter_widths=[3, 5, 3], causal=True, channels=128)),
    (vp.TemporalModel, dict(filter_widths=[3, 3], dense=True, channels=64)),
    (vp.TemporalModelOptimized1f, dict(filter_widths=[3, 3, 3, 3, 3], causal=False)),
    (vp.TemporalModelOptimized1f, dict(filter_widths=[3, 3, 3], causal=True, channels=256)),
])
def test_module_contract(cls, kw):
    """Key set / order / shapes of the state_dict (SURVEY.md §8b) and the derived attributes."""
    from oracle import temporal_model_oracle as orc
    m = cls(17, 2, 17, **kw)
    C = kw.get("channels", 1024)
    fw = kw["filter_widths"]
    nb = len(fw) - 1
    strided = cls is vp.TemporalModelOptimized1f
    a = orc.arch(fw, causal=kw.get("causal", False), dense=kw.get("dense", False), strided=strided)
    keys = list(m.state_dict().keys())
    bn = lambda p: [f"{p}.weight", f"{p}.bias", f"{p}.running_mean", f"{p}.running_var",
                    f"{p}.num_batches_tracked"]
    expect = bn("expand_bn") + ["shrink.weight", "shrink.bias", "expand_conv.weight"] + \
        [f"layers_conv.{i}.weight" for i in range(2 * nb)] + \
        sum((bn(f"layers_bn.{i}") for i in range(2 * nb)), [])
    assert keys == expect
    sd = m.state_dict()
    assert tuple(sd["expand_conv.weight"].shape) == (C, 34, fw[0])
    assert tuple(sd["shrink.weight"].shape) == (51, C, 1) and tuple(sd["shrink.bias"].shape) == (51,)
    for i in range(nb):
        assert tuple(sd[f"layers_conv.{2 * i}.weight"].shape) == (C, C, a["taps"][i + 1])
        assert tuple(sd[f"layers_conv.{2 * i + 1}.weight"].shape) == (C, C, 1)
    assert sd["expand_bn.num_batches_tracked"].dtype == torch.int64
    assert m.pad == a["pad"] and m.causal_shift == a["shift"]
    assert m.receptive_field() == a["receptive_field"]
    assert isinstance(m.drop, torch.nn.Dropout) and isinstance(m.relu, torch.nn.ReLU)
    m.set_bn_momentum(0.03)
    assert m.expand_bn.momentum == 0.03 and all(b.momentum == 0.03 for b in m.layers_bn)
    # the oracle's seeded parameters load into the module (same layout as the reference's)
    m.load_state_dict(orc.make_state_dict(17, 2, 17, fw, C, dense=kw.get("dense", False)))


def test_no_cpu_fallback():
    m = vp.TemporalModel(17, 2, 17, [3, 3, 3], channels=64).eval()
    with pytest.raises(AssertionError):
        m(torch.zeros(2, 27, 17, 3))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.zeros(2, 27, 17, 2))
    with pytest.raises(AssertionError, match="odd filter widths"):
        vp.TemporalModelOptimized1f(17, 2, 17, [3, 2])


def test_fused_losses_refuse_cpu_tensors():
    """The loss head is CUDA-only (no torch-op fallback): CPU tensors raise."""
    from videopose3d_b200 import loss as vloss
    pred = torch.randn(4, 1, 17, 3)
    with pytest.raises(RuntimeError):
        vloss.bone_length_penalty(pred, 2, [-1] + list(range(16)))
    with pytest.raises(RuntimeError):
        vloss.mpjpe(pred, pred.clone())


def test_copies_and_replicas_start_with_empty_engine_state():
    """copy / deepcopy / pickle / DataParallel replicas start with empty engine states of their own
    (a collected copy used to destroy the original's plans), and deepcopy works after a forward
    has created ctypes handles (EMA / best-model patterns)."""
    import copy
    import pickle
    from videopose3d_b200.temporal_model import _EngineState
    m = vp.TemporalModelOptimized1f(17, 2, 17, [3, 3], channels=64)
    destroyed = []
    m._engine._finalizer.detach()
    m._engine = engine = _EngineState()
    engine._finalizer.detach()
    # what a first forward leaves behind
    plan = engine.last = engine.add((0, "fp16"), _capi.ctypes.c_void_p(1234))
    plan.eval = plan.train = plan.expand_t = "versions"
    clones = [copy.deepcopy(m), copy.copy(m), pickle.loads(pickle.dumps(m)),
              m._replicate_for_data_parallel()]
    for c in clones:
        assert isinstance(c._engine, _EngineState) and c._engine is not engine
        assert c._engine.plans == {} and c._plan is None
        assert sorted(c.state_dict()) == sorted(m.state_dict())
    assert torch.equal(clones[0].shrink.weight, m.shrink.weight)
    assert clones[0].shrink.weight.data_ptr() != m.shrink.weight.data_ptr()
    del clones
    assert len(engine.plans) == 1 and destroyed == []      # the original still owns its plan
    assert m.invalidate() is m
    assert (plan.eval, plan.train, plan.expand_t) == (None, None, None)


def test_training_operator_entries_validate_before_launching():
    """vp3d_wgrad_gemm and the BatchNorm-pass entries report bad arguments without touching a device
    (the pointers below are never dereferenced)."""
    ct = _capi.ctypes
    lib = _capi.load()
    assert lib.vp3d_wgrad_gemm(None, None) == -1
    d = _capi.WgradDesc()
    fake = 1 << 20
    d.dz = d.x = d.grad = d.partial = fake
    d.dz_ld = d.x_ld = 256
    d.planes, d.rows, d.taps, d.taps_out = 1, 1000, 3, 3
    d.c_out = d.c_in = d.c_in_cols = 256
    d.tap_col_step = 256
    d.partial_bytes = 3 * 256 * 256 * 4 - 4          # one float short of a single split
    assert lib.vp3d_wgrad_gemm(ct.byref(d), None) == -4
    assert b"partial buffer too small" in lib.vp3d_last_error()
    d.planes = 3
    assert lib.vp3d_wgrad_gemm(ct.byref(d), None) == -1
    d.planes, d.merged = 1, 1                          # merged needs taps == 1
    assert lib.vp3d_wgrad_gemm(ct.byref(d), None) == -1
    c = 8256
    args = [fake, 4, 0, 100, 0, fake, fake, None, None, 0.1, 1e-5, fake, fake, fake, fake, c, c,
            fake, 96 * c, fake, (c + 31) // 32, None]
    assert lib.vp3d_bn_stats_finalize(*args) == -2     # more than 8192 channels
    args[15] = args[16] = 1024
    args[18] = 96 * 1024 - 1                           # scratch one float short
    assert lib.vp3d_bn_stats_finalize(*args) == -4
    assert lib.vp3d_ordered_col_sums(fake, 10, 3, 64, 64, 1, None, None, fake, fake, fake, 64 * 64,
                                     fake, 2, None) == -1
    assert lib.vp3d_bn_apply(fake, 0, fake, 0, 1, 10, 100, fake, fake, 0.0, 0, 0, None, 0, 0, 0, 0,
                             0, None) == -1            # channels not a multiple of 64
    assert lib.vp3d_bn_bwd_apply(fake, 0, fake, 0, fake, 0, 1, 10, 64, fake, fake, None, None, 0.0,
                                 0, 0, None, None, None, 64, 0, None) == -1   # sums needed unless frozen


@pytest.mark.parametrize("precision,changes,code,word", [
    # fp16 (and int8, whose residual and 16-bit output are fp16): one plane, inference only
    ("fp16", dict(a_planes=2), -1, b"single-plane"),
    ("fp16", dict(out_planes=2), -1, b"single-plane"),
    ("fp16", dict(stats=1 << 20), -1, b"inference-only"),
    ("int8", dict(bnb_z=1 << 20), -1, b"inference-only"),
    # int8 k-blocks are 128 one-byte elements, and taps step rows
    ("int8", dict(k_per_tap=64), -1, b"k_per_tap"),
    ("int8", dict(tap_col_step=128), -1, b"tap_col_step"),
    # a u8 output: fp16 or int8, 16-byte aligned rows covering n_pad
    ("bf16", dict(res=None, out_u8=1 << 20), -1, b"u8 output"),
    ("int8", dict(out_u8_ld=48), -1, b"out_u8_ld"),
    ("int8", dict(out_u8_ld=72), -1, b"out_u8_ld"),
    ("int8", dict(out_u8=(1 << 20) + 8), -1, b"aligned"),
    # int8 / u8 launches are affine + ReLU [+ a one-plane residual over every column]
    ("int8", dict(relu=0), -2, b"affine + ReLU"),
    ("int8", dict(shift=None), -2, b"affine + ReLU"),
    ("int8", dict(out_f32=1 << 20), -2, b"affine + ReLU"),
    ("int8", dict(res_col_begin=64), -2, b"every column"),
    ("int8", dict(res_cols=64), -2, b"every column"),
    ("int8", dict(res_planes=2), -2, b"one-plane residual"),
    # int8 writes u8 alone, or with a residual fp16 [+ u8]; fp16 + u8 has no residual
    ("int8", dict(out=None), -2, b"with a residual, fp16"),
    ("int8", dict(res=None), -2, b"int8 writes u8 alone"),
    ("int8", dict(res=None, out_u8=None), -2, b"int8 writes u8 alone"),
    ("fp16", dict(), -2, b"without a residual"),
    ("fp16", dict(res=None, out=None), -2, b"fp16 without a residual writes fp16 + u8"),
])
def test_conv_gemm_rejects_unsupported_int8_u8_fp16_launches(precision, changes, code, word):
    """vp3d_conv_gemm checks every int8 / u8 / fp16 condition before touching a device (the pointers
    below are never dereferenced)."""
    ct = _capi.ctypes
    lib = _capi.load()
    fake = 1 << 20
    d = _capi.ConvDesc()
    d.a = d.w = d.scale = d.shift = d.res = d.out = d.out_u8 = fake
    d.samples, d.a_rows, d.a_ld, d.taps, d.k_per_tap, d.n_pad = 1, 130, 128, 3, 128, 128
    d.per_sample_tiles, d.tap_row_step, d.out_rows = 1, 1, 128
    d.precision = {"bf16": 0, "fp16": 3, "int8": 4}[precision]
    d.relu = 1
    d.res_ld = d.out_ld = d.out_u8_ld = 128
    d.res_rows_per_sample, d.res_row_step, d.res_row_off = 130, 1, 1
    for k, v in changes.items():
        assert k in dict(d._fields_)
        setattr(d, k, v)
    assert lib.vp3d_conv_gemm(ct.byref(d), None) == code
    assert word in lib.vp3d_last_error()
