"""The backward routes that tests/test_hrnet_grad_gpu.py covers at the real HRNet widths, recorded on the CPU.

One training step of HRNet-w32 and -w48 at 2x3x256x192 runs through the launch recorder of
tests/golden/make_dispatch_trace.py (no GPU, nothing computed). The step must still take the routes the small golden
HRNet never reaches: the chunked tensor-core weight gradient, CUDA-core weight gradients at stride 1 and at stride 2
(compact dY), and tensor-core convolutions with 384 input channels. If a routing change stops sending work down one of
them, the GPU tests would no longer cover it; this test fails instead. It asserts which kinds of launch occur, not a
golden trace (tests/test_conv_dispatch_cpu.py pins that for the small configurations).
"""
import collections
import importlib.util
import os

import pytest

_spec = importlib.util.spec_from_file_location(
    "make_dispatch_trace", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_dispatch_trace.py"))
T = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(T)

# position of B in a recorded launch ([name, *arguments], include/fpd_b200.h); H, W, Cin, Cout, k follow, and for the
# CUDA-core convolutions the stride after them
_B_AT = {"fpd_conv2d_wgrad_tc_fused": 10, "fpd_conv2d_simt_wgrad": 5, "fpd_conv2d_simt_fwd": 6, "fpd_conv2d_tc_h": 15,
         "fpd_conv2d_tc_h_stats": 13}
Shape = collections.namedtuple("Shape", ("B", "H", "W", "Cin", "Cout", "k", "stride"))


def _shapes(calls, name):
    i = _B_AT[name]
    return [Shape(*c[i:i + 6], c[i + 6] if "simt" in name else 1) for c in calls if c[0] == name]


def _hrnet(width):
    def make():
        from bench import hrnet_cfg
        from fpd_b200.lib.models import pose_hrnet as H
        return H.get_pose_net(hrnet_cfg(width), False), (2, 3, 256, 192)
    return make


def _train_step(width, monkeypatch):
    """-> (recorded launches of one fp32 training step, the calls of ops.conv2d_wgrad_tc_chunked and the number of
    launches each made)."""
    import fpd_b200  # noqa: F401
    from fpd_b200 import ops
    name = "hrnet_w%d" % width
    monkeypatch.setitem(T.NETS, name, _hrnet(width))
    chunked = []
    fused_calls = [0]
    chunked_fn, fused_fn = ops.conv2d_wgrad_tc_chunked, ops.conv2d_wgrad_tc_fused

    def fused(*args, **kw):
        fused_calls[0] += 1
        return fused_fn(*args, **kw)

    def chunked_spy(x, dy, ksize, chunks, **kw):
        n0 = fused_calls[0]
        dw = chunked_fn(x, dy, ksize, chunks, **kw)
        chunked.append((Shape(*x.shape, dy.shape[3], ksize, 1), tuple(chunks), fused_calls[0] - n0))
        return dw
    monkeypatch.setattr(ops, "conv2d_wgrad_tc_fused", fused)
    monkeypatch.setattr(ops, "conv2d_wgrad_tc_chunked", chunked_spy)
    return T.trace("%s/train_fp32/default" % name), chunked


@pytest.mark.parametrize("width", [32, 48])
def test_training_step_takes_the_wide_routes(width, monkeypatch):
    calls, chunked = _train_step(width, monkeypatch)
    wgrad = _shapes(calls, "fpd_conv2d_wgrad_tc_fused")
    assert wgrad and all(s.B == 2 and s.k in (1, 3) for s in wgrad)     # the argument positions are the ABI's
    # ---- chunked tensor-core weight gradients: one launch per (Cin chunk, Cout chunk), split along Cin
    assert all(n == (s.Cin // ci) * (s.Cout // co) for s, (ci, co), n in chunked), chunked
    split_cin = [(s, ch) for s, ch, _ in chunked if ch[0] < s.Cin and s.k == 3]
    assert split_cin, "no 3x3 weight gradient is split along its input channels"
    top = 8 * width                                        # branch 3's width, at 8x6
    assert any((s.H, s.W, s.Cin, s.Cout) == (8, 6, top, top) for s, _ in split_cin), split_cin
    if width == 48:
        # 384 -> 384: split along both channel axes
        assert any(ch[0] < s.Cin and ch[1] < s.Cout and s.Cin == top for s, ch, _ in chunked), chunked
    launched = sum(n for _, _, n in chunked)
    assert 0 < launched <= len(wgrad)
    # ---- tensor-core forward and data-gradient convolutions at branch 3's width (w48: 384 input channels, three
    # 128-column output slices)
    tc = _shapes(calls, "fpd_conv2d_tc_h") + _shapes(calls, "fpd_conv2d_tc_h_stats")
    assert any(s.Cin == top and s.Cout == top and s.k == 3 for s in tc)
    simt = _shapes(calls, "fpd_conv2d_simt_wgrad")
    if width == 48:
        # ---- w48: CUDA-core weight gradients at stride 1 (branch 0's 48 -> 48 3x3s) and at stride 2
        s1 = [s for s in simt if s.k == 3 and s.stride == 1]
        s2 = [s for s in simt if s.k == 3 and s.stride == 2]
        assert any((s.H, s.W, s.Cin, s.Cout) == (64, 48, 48, 48) for s in s1), s1
        assert s2, simt
        # the stride-2 convolutions ran forward at stride 1 on the tensor cores: their weight gradients took the compact
        # dY of Engine._conv_at's CUDA-core branch
        assert not [s for s in _shapes(calls, "fpd_conv2d_simt_fwd") if s.stride == 2]
    print("hrnet w%d: %d tensor-core weight-gradient launches, %d of them from %d chunked calls; %d CUDA-core weight "
          "gradients (%d 3x3 at stride 1, %d at stride 2); %d tensor-core convolutions with Cin = %d" % (
              width, len(wgrad), launched, len(chunked), len(simt),
              sum(s.k == 3 and s.stride == 1 for s in simt), sum(s.k == 3 and s.stride == 2 for s in simt),
              sum(s.Cin == top for s in tc), top))
