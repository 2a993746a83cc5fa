"""CPU: the host side of int8 streaming sessions (model.streaming(..., int8=True),
VP3D_STREAM_INT8) -- the ring bytes of the u8 history, the flag's C-ABI checks that run before any
device work, and the validation streaming() applies before it touches a device."""
import pytest

import videopose3d_b200 as vp
from videopose3d_b200 import _capi, streaming


@pytest.mark.parametrize("fw,C", [([3, 3, 3], 64), ([3, 3, 3, 3, 3], 1024), ([3, 5, 3], 100)])
@pytest.mark.parametrize("augment", [False, True])
@pytest.mark.parametrize("provisional", [False, True])
def test_ring_bytes_int8(fw, C, augment, provisional):
    """int8 adds, per ring of a residual block, one byte per (padded) channel and frame position of
    the 16-bit rings (both mirror halves, twice with augment); ring 0 is unchanged."""
    m = vp.TemporalModel(17, 2, 17, fw, channels=C)
    K = 3
    plain = streaming.ring_bytes_per_stream(m, K, augment=augment, provisional=provisional)
    q = streaming.ring_bytes_per_stream(m, K, augment=augment, provisional=provisional, int8=True)
    tail = streaming.lookahead(m) if provisional else 0
    c = -(-C // 64) * 64
    extra = sum(2 * (h + K + tail + 1) * c for h in streaming.ring_history(fw)[1:])
    assert q - plain == (2 if augment else 1) * extra
    # the 16-bit ring bytes of the residual blocks, halved: q adds about half the 16-bit figure
    blocks = sum(2 * (h + K + tail + 1) * c * 2 for h in streaming.ring_history(fw)[1:])
    assert 2 * extra == blocks


def test_int8_ring_bytes_of_the_bench_arc():
    """Arc 3,3,3,3,3 at C = 1024, K = 1: about 1.5 MB instead of 1.0 MB per stream."""
    m = vp.TemporalModel(17, 2, 17, [3, 3, 3, 3, 3], channels=1024)
    plain = streaming.ring_bytes_per_stream(m, 1)
    q = streaming.ring_bytes_per_stream(m, 1, int8=True)
    assert 0.95e6 < plain < 1.05e6
    assert 1.45 < q / plain < 1.5


def test_int8_flag_c_abi_without_gpu():
    lib = _capi.load()
    fake = 1 << 20   # never dereferenced: the checks fail first
    flag = _capi.VP3D_STREAM_INT8
    assert flag == 16
    aug, prov = _capi.VP3D_STREAM_AUGMENT, _capi.VP3D_STREAM_PROVISIONAL
    for flags in (flag, flag | aug, flag | prov, flag | aug | prov):
        assert lib.vp3d_stream_state_bytes_ex(None, 4, 1, flags) == 0
    for flags in (flag, flag | prov):
        # the flag passes the flag check (the null plan is reported next)
        assert lib.vp3d_stream_init_ex(None, fake, 1 << 20, 4, 1, flags, None, None, None) == -1
        assert b"null plan" in lib.vp3d_last_error()
    for flags in (flag | 2, flag | 8, flag | 32):
        assert lib.vp3d_stream_init_ex(fake, fake, 1 << 20, 4, 1, flags, None, None, None) == -1
        assert b"unknown flags" in lib.vp3d_last_error()


def test_streaming_int8_argument_checks_without_gpu():
    m = vp.TemporalModel(17, 2, 17, [3, 3], channels=64).eval()
    for precision in ("fp16", "bf16", "bf16x3"):
        m.set_precision(precision)
        with pytest.raises(ValueError, match="int8"):
            m.streaming(2, 1, int8=True)
    # an int8 model without the keyword: refused, pointing at it
    m.set_precision("int8")
    with pytest.raises(NotImplementedError, match="int8=True"):
        m.streaming(2, 1)
    # with it, the CPU model is refused before any device work
    with pytest.raises(RuntimeError, match="CUDA device"):
        m.streaming(2, 1, int8=True)
    with pytest.raises(RuntimeError, match="CUDA device"):
        m.streaming(2, 1, int8=True, provisional=True)
