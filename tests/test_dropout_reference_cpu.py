"""CPU: the dropout mask restated in Python (oracle/train_emulation.dropout_mask) and the masked
references built on it.

The training kernels draw their dropout masks from a counter hash of (seed, layer, element), so a
training step with dropout can be replayed exactly: the fp64 reference is forward_torch with the same
masks multiplied in (autograd gives its gradients), and the quantisation-aware emulation
train_step(masks=...) must agree with it when it rounds nothing (planes = 0)."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import temporal_model_oracle as orc
from oracle import train_emulation as emu


def _reference_step(sd, x, gy, fw, causal, dilated, momentum, masks):
    """float64 autograd through forward_torch(masks=...): y, gradients, new running statistics."""
    sd = {k: v.double().clone() if v.is_floating_point() else v.clone() for k, v in sd.items()}
    leaves = {k: v.requires_grad_(True) for k, v in sd.items()
              if v.is_floating_point() and "running_" not in k}
    y = orc.forward_torch(sd, x.double(), fw, causal=causal, strided=not dilated, training=True,
                          momentum=momentum, update_stats=True, masks=masks)
    (y * gy.double()).sum().backward()
    grads = {k: v.grad for k, v in leaves.items()}
    stats = {k: v for k, v in sd.items() if "running_" in k}
    return y.detach(), grads, stats


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-300))


@pytest.mark.parametrize("name", ["opt_333_c128_train", "opt_35_c128_train_causal",
                                  "opt_33_c40_train", "tm_333_c128_train"])
def test_masked_emulation_equals_fp64_autograd(name):
    """train_step(planes=0, masks) == autograd of the masked forward, for every output: y, each
    parameter gradient and each updated running statistic, strided and dilated, C = 40 padded to 64."""
    meta, sd, x, _, new = load_golden(name)
    dilated = meta["cls"] == "TemporalModel"
    N, T = x.shape[0], x.shape[1]
    masks = emu.model_masks(emu.step_seed(7), meta["fw"], N, T, meta["C"], 0.25, dilated=dilated)
    gy = torch.from_numpy(new["gy"])
    out = emu.train_step(sd, x, gy, meta["fw"], causal=meta["causal"], planes=0,
                         momentum=meta["momentum"], dilated=dilated, masks=masks)
    y, grads, stats = _reference_step(sd, x, gy, meta["fw"], meta["causal"], dilated,
                                      meta["momentum"], masks)
    assert out["y"].shape == y.shape
    assert _rel(out["y"], y) <= 1e-10
    assert set(out["grads"]) == set(grads)
    for k, g in grads.items():
        assert _rel(out["grads"][k], g) <= 1e-10, k
    assert set(out["new_stats"]) == set(stats)
    for k, v in stats.items():
        assert _rel(out["new_stats"][k], v) <= 1e-10, k
    # the masks change the step (they are not silently ignored by either side)
    plain = emu.train_step(sd, x, gy, meta["fw"], causal=meta["causal"], planes=0,
                           momentum=meta["momentum"], dilated=dilated)
    assert _rel(plain["y"], y) > 1e-2


def test_unmasked_dilated_emulation_equals_fp64_autograd():
    """Without masks the dilated emulation is the plain fp64 training step of TemporalModel."""
    meta, sd, x, _, new = load_golden("tm_35_c128_train_causal")
    gy = torch.from_numpy(new["gy"])
    out = emu.train_step(sd, x, gy, meta["fw"], causal=True, planes=0, momentum=meta["momentum"],
                         dilated=True)
    y, grads, stats = _reference_step(sd, x, gy, meta["fw"], True, True, meta["momentum"], None)
    assert _rel(out["y"], y) <= 1e-10
    for k, g in grads.items():
        assert _rel(out["grads"][k], g) <= 1e-10, k
    for k, v in stats.items():
        assert _rel(out["new_stats"][k], v) <= 1e-10, k


def _u16(seed, layer, e):
    """Straight-line restatement of the hash for single elements (Python ints, explicit wrapping)."""
    U = 0xFFFFFFFF
    P = e >> 1
    key = (seed & U) ^ (((seed >> 32) * 0x7F4A7C15) & U) ^ ((layer * 0x632BE5AB) & U) ^ \
        (((P >> 32) * 0x85EBCA77) & U)
    h = ((P & U) * 0x9E3779B1 + key) & U
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & U
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & U
    h ^= h >> 16
    return (h >> 16) if e & 1 else (h & 0xFFFF)


SEED = 0x2F3A_1B7C_9D40_5E61   # high word nonzero


def test_mask_values_and_keep_rate():
    p, rows, c = 0.25, 1000, 128
    m = emu.dropout_mask(SEED, 3, rows, c, c, p).numpy()
    assert m.shape == (rows, c) and m.dtype == np.float64
    inv_keep = float(np.float32(1) / (np.float32(1) - np.float32(p)))
    assert set(np.unique(m)) == {0.0, inv_keep}
    rate = float((m != 0).mean())
    sigma = (p * (1 - p) / m.size) ** 0.5
    assert abs(rate - (1 - p)) <= 3 * sigma, rate


def test_mask_matches_scalar_hash_including_high_pair_words():
    """The vectorised mask against the scalar restatement, at element indices beyond 2^33 too
    (where the pair index's high word enters the key)."""
    p = 0.25
    thresh = int(np.float32(p) * 65536)
    m = emu.dropout_mask(SEED, 5, 40, 64, 64, p).numpy()
    for r, ch in [(0, 0), (0, 1), (3, 17), (39, 63), (21, 32)]:
        assert (m[r, ch] != 0) == (_u16(SEED, 5, r * 64 + ch) >= thresh)
    c_pad = 1 << 32                                         # row r starts at element r * 2^32
    mb = emu.dropout_mask(SEED, 5, 6, 40, c_pad, p).numpy()
    for r in range(6):
        for ch in range(40):
            assert (mb[r, ch] != 0) == (_u16(SEED, 5, r * c_pad + ch) >= thresh), (r, ch)
    assert not np.array_equal(mb[2], mb[4])                 # rows differing only in P >> 32


def test_mask_threshold_is_truncated():
    """p = 0.1: fp32(p) * 65536 = 6553.6 -> the kernels compare against 6553, not 6554."""
    p, rows, c = 0.1, 1000, 64
    m = emu.dropout_mask(SEED, 2, rows, c, c, p).numpy()
    u = np.array([_u16(SEED, 2, e) for e in range(rows * c)]).reshape(rows, c)
    assert ((u >= 6553) == (m != 0)).all()
    assert (u == 6553).any(), "the fixture must contain the boundary value"
    inv_keep = float(np.float32(1) / (np.float32(1) - np.float32(0.1)))
    assert inv_keep != 1 / 0.9 and set(np.unique(m)) == {0.0, inv_keep}


def test_even_and_odd_elements_read_different_halves():
    p, rows, c = 0.5, 512, 64
    m = emu.dropout_mask(SEED, 2, rows, c, c, p).numpy() != 0
    even, odd = m[:, 0::2], m[:, 1::2]
    # halves of one hash are independent: the pair's two decisions agree about half of the time
    agree = float((even == odd).mean())
    assert abs(agree - 0.5) < 0.05, agree
    for r, ch in [(0, 0), (7, 9), (100, 62)]:
        assert m[r, ch] == (_u16(SEED, 2, r * c + ch) >= 32768)


def test_layers_and_seeds_give_different_masks():
    p, rows, c = 0.25, 256, 128
    base = emu.dropout_mask(SEED, 1, rows, c, c, p).numpy() != 0
    for other in (emu.dropout_mask(SEED, 2, rows, c, c, p), emu.dropout_mask(SEED + 1, 1, rows, c, c, p),
                  emu.dropout_mask(SEED ^ (1 << 40), 1, rows, c, c, p)):
        diff = float(((other.numpy() != 0) != base).mean())
        assert abs(diff - 2 * p * (1 - p)) < 0.03, diff     # independent masks differ 37.5 % of the time


def test_padded_channels_change_the_index():
    """C = 100 on a plan padded to 128: row r, channel ch is element r * 128 + ch, not r * 100 + ch."""
    p, rows = 0.25, 64
    padded = emu.dropout_mask(SEED, 4, rows, 100, 128, p)
    dense = emu.dropout_mask(SEED, 4, rows, 100, 100, p)
    full = emu.dropout_mask(SEED, 4, rows, 128, 128, p)
    assert torch.equal(padded, full[:, :100])
    assert torch.equal(padded[0], dense[0])                 # row 0 is the same either way
    assert not torch.equal(padded[1:], dense[1:])
    flat = emu.dropout_mask(SEED, 4, 1, rows * 128, rows * 128, p).reshape(rows, 128)
    assert torch.equal(padded, flat[:, :100])


def test_model_masks_layer_numbering_and_rows():
    fw, N, T, C = [3, 3, 3], 4, 34, 40
    ms = emu.model_masks(SEED, fw, N, T, C, 0.25, dilated=True)
    L = emu.layer_lengths(fw, T, dilated=True)
    assert L == [32, 26, 8]
    assert sorted(ms) == [0, 1, 2, 3, 4]
    for layer, m in ms.items():
        assert tuple(m.shape) == (N * L[(layer + 1) // 2], C)
        assert torch.equal(m, emu.dropout_mask(SEED, layer, m.shape[0], C, 64, 0.25))
    assert emu.layer_lengths([3, 5], 15) == [5, 1]
