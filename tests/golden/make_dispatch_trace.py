"""Generate tests/golden/dispatch_trace.json.gz: the native launches the engine issues for one step of each network and
precision setting, recorded on the CPU without a GPU:

    python tests/golden/make_dispatch_trace.py

Engine.forward / Engine.backward run on CPU tensors with _native.lib() replaced by a recorder. Planner and query symbols
(*_supported, *_kernel, *_plan, *_blocks, *_workspace_bytes, fpd_set_*) go to the real library, which loads and plans
without a device; every other symbol is recorded as its name, its int and float arguments and whether each pointer is
null, and returns 0. Nothing is computed, so the trace pins which kernel every convolution runs on, with which operand
forms, statistics and scales, and in which order; tests/test_conv_dispatch_cpu.py checks it.

The planners answer for 132 SMs: an H100 SXM, or no device at all.
"""
import ctypes
import gzip
import io
import json
import os
import sys
import types

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "dispatch_trace.json.gz")
NS = types.SimpleNamespace
SM_COUNT = 132
_QUERY_SUFFIXES = ("_supported", "_kernel", "_plan", "_blocks", "_workspace_bytes")
_QUERY_NAMES = ("fpd_last_error", "fpd_version", "fpd_sm_count", "fpd_launch_count")


class _Recorder:
    def __init__(self, lib):
        self._lib = lib
        self.calls = []

    def __getattr__(self, name):
        if name in _QUERY_NAMES or name.startswith("fpd_set_") or name.endswith(_QUERY_SUFFIXES):
            return getattr(self._lib, name)

        def launch(*args):
            self.calls.append([name] + [_arg(a) for a in args])
            return 0
        return launch


def _arg(a):
    if a is None:
        return "null"
    if isinstance(a, ctypes.c_void_p):
        return "ptr" if a.value else "null"
    if isinstance(a, ctypes.Array):   # pointer arrays read back as ints (or None)
        return [("ptr" if v else "null") if a._type_ is ctypes.c_void_p else v for v in a]
    if isinstance(a, bool):
        return int(a)
    if isinstance(a, (int, float)):
        return a
    raise TypeError("unexpected argument %r" % (a,))


def _hourglass():
    from fpd_b200.lib.models import hourglass as H
    cfg = NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=64, NUM_STACKS=2, NUM_BLOCKS=1), NUM_JOINTS=16))
    return H.get_pose_net(cfg, False), (2, 3, 64, 64)


def _hrnet():
    from fpd_b200.lib.models import pose_hrnet as H

    class Cfg(dict):
        __getattr__ = dict.__getitem__

    def wrap(d):
        return Cfg({k: wrap(v) for k, v in d.items()}) if isinstance(d, dict) else d

    def stage(nmod, chans):
        return dict(NUM_MODULES=nmod, NUM_BRANCHES=len(chans), BLOCK='BASIC', NUM_BLOCKS=[1] * len(chans),
                    NUM_CHANNELS=chans, FUSE_METHOD='SUM')
    cfg = wrap(dict(MODEL=dict(NUM_JOINTS=17, INIT_WEIGHTS=False, PRETRAINED='', EXTRA=dict(
        PRETRAINED_LAYERS=['*'], FINAL_CONV_KERNEL=1, STAGE2=stage(1, [16, 32]), STAGE3=stage(1, [16, 32, 64]),
        STAGE4=stage(1, [16, 32, 64, 128])))))
    return H.get_pose_net(cfg, is_train=False), (2, 3, 64, 48)


def _resnet():
    from fpd_b200.lib.models import pose_resnet as R
    cfg = NS(MODEL=NS(NUM_JOINTS=17, INIT_WEIGHTS=False, PRETRAINED='', EXTRA=NS(
        NUM_LAYERS=18, DECONV_WITH_BIAS=True, NUM_DECONV_LAYERS=3, NUM_DECONV_FILTERS=[64, 32, 32],
        NUM_DECONV_KERNELS=[4, 3, 2], FINAL_CONV_KERNEL=1)))
    return R.get_pose_net(cfg, is_train=False), (2, 3, 64, 64)


NETS = {"hourglass": _hourglass, "hrnet": _hrnet, "resnet": _resnet}

# mode: (training precision, inference precision, training, record_tape)
MODES = {"train_fp32": ("fp32", "fp32", True, True), "train_fp16": ("fp16", "fp32", True, True),
         "eval_tape_fp16": ("fp16", "fp32", False, True),
         "infer_fp32": ("fp32", "fp32", False, False), "infer_fp16": ("fp32", "fp16", False, False)}

# option: (module, attribute, value) patches, or ("env", name, value)
OPTIONS = {"default": [], "tf32": [("env", "FPD_PRECISION", "tf32")],
           "no_conv_h": [("ops", "CONV_H", False)], "no_conv_f16": [("ops", "CONV_F16", False)],
           "no_conv_f16_dgrad": [("ops", "CONV_F16_DGRAD", False)], "no_fused_reduce": [("ops", "FUSED_REDUCE", False)],
           "conv_stats_0": [("ops", "CONV_STATS", "0")], "conv_stats_1": [("ops", "CONV_STATS", "1")],
           "no_stride2_tc": [("engine", "STRIDE2_TC", False)]}

CASES = ["%s/%s/%s" % (n, m, o) for n in NETS for o in OPTIONS for m in MODES
         if o == "default" or m in ("train_fp32", "train_fp16", "infer_fp32", "infer_fp16")]


def trace(case):
    """-> the recorded launches of one forward (and, with a tape, backward) of case "net/mode/option"."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native, engine, ops
    net_name, mode, option = case.split("/")
    tprec, iprec, training, tape = MODES[mode]
    with pytest.MonkeyPatch.context() as mp:
        for mod, attr, value in OPTIONS[option]:
            if mod == "env":
                mp.setenv(attr, value)
            else:
                mp.setattr({"ops": ops, "engine": engine}[mod], attr, value)
        rec = _Recorder(_native.lib())
        mp.setattr(_native, "lib", lambda: rec)
        mp.setattr(ops, "_stream", lambda: ctypes.c_void_p(0))
        mp.setattr(ops, "_chk", lambda t, name: None)
        mp.setattr(ops._ws, "get", lambda nbytes, device: torch.empty(max(int(nbytes), 1), dtype=torch.uint8))
        mp.setattr(ops, "_counter", lambda device: torch.zeros(16, dtype=torch.int32))
        torch.manual_seed(0)
        net, shape = NETS[net_name]()
        net.train(training)
        eng = net.engine()
        eng.training_precision, eng.inference_precision = tprec, iprec
        img = torch.zeros(shape)
        with torch.no_grad():
            ctx = eng.forward(img, training, tape)
            if tape:
                eng.backward(ctx, [torch.zeros_like(v.data) for v in ctx.outs])
    return rec.calls


def trace_all():
    return {case: trace(case) for case in CASES}


def dumps(traces):
    """The fixture's bytes: sorted JSON, gzip without a time stamp or file name (the same traces give the same file)."""
    buf = io.BytesIO()
    with gzip.GzipFile(filename="", mode="wb", fileobj=buf, mtime=0) as f:
        f.write(json.dumps(traces, sort_keys=True, separators=(",", ":")).encode())
    return buf.getvalue()


def load():
    with gzip.open(OUT, "rb") as f:
        return json.loads(f.read())


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    from fpd_b200 import _native
    assert _native.lib().fpd_sm_count() == SM_COUNT, "the fixture is recorded for %d SMs" % SM_COUNT
    data = dumps(trace_all())
    with open(OUT, "wb") as f:
        f.write(data)
    print("%s: %d cases, %d bytes" % (OUT, len(CASES), len(data)))
