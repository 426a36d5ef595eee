"""CPU suite: the C-ABI library loads and exports every symbol include/fpd_b200.h declares (no compute calls)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "fpd_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(fpd_[a-z0-9_]+)\s*\(", src)) - {"fpd_stream_t"})


def test_library_exports_every_declared_symbol():
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    assert os.path.exists(N.LIB_PATH), "build the library first: python -c 'import __graft_entry__ as g; g.build()'"
    h = ctypes.CDLL(N.LIB_PATH)
    declared = _declared_symbols()
    assert len(declared) >= 35
    for name in declared:
        assert hasattr(h, name), "missing export: " + name
    # the ctypes table covers the whole header and nothing else
    assert sorted(N.EXPORTED_SYMBOLS) == declared
    assert N.lib().fpd_version() >= 100
    assert N.lib().fpd_conv2d_tc_ts_supported(64, 64, 3) == 1
    assert N.lib().fpd_conv2d_tc_ts_supported(3, 32, 7) == 0


def test_missing_library_fails_loudly(tmp_path, monkeypatch):
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    monkeypatch.setattr(N, "_lib", None)
    monkeypatch.setattr(N, "LIB_PATH", str(tmp_path / "nope.so"))
    import pytest
    with pytest.raises(N.NativeLibraryMissing):
        N.lib()


def test_every_host_module_imports_on_cpu():
    """Import (= byte-compile) every Python module of the package and the top-level scripts: no GPU needed."""
    import importlib
    import fpd_b200  # noqa: F401
    for name in ("_native", "ops", "engine", "engine_hrnet", "autograd_bridge", "train_step", "infer_step", "parallel",
                 "dropin", "targets",
                 "lib.models.hourglass", "lib.models.pose_hrnet", "lib.core.loss", "lib.core.function",
                 "lib.core.inference", "lib.core.evaluate", "lib.utils.transforms", "lib.nms.nms"):
        importlib.import_module("fpd_b200." + name)
    import ast
    for script in ("bench.py", "__graft_entry__.py", "tools/profile_step.py", "tools/profile_convs.py",
                   "tools/diag_net.py", "tools/diag_grad.py", "tools/diag_resnet_head.py", "tools/cpu_thread_sweep.py",
                   "tools/timeline_step.py"):
        ast.parse(open(os.path.join(ROOT, script)).read(), script)


def test_kernel_shape_planners_on_cpu():
    """The support predicates of the wgmma convolution and weight-gradient kernels are pure host code: every shape of
    the BASELINE configs must be taken, the documented exceptions not."""
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    lib = N.lib()
    # hourglass student (64/128 ch) and teacher (128/256 ch) convolutions at every level, both operand encodings
    for hw in (64, 32, 16, 8, 4):
        for (cin, cout, k) in ((64, 64, 3), (128, 128, 3), (128, 64, 1), (64, 128, 1), (256, 128, 1), (128, 256, 1),
                               (256, 256, 1), (256, 16, 1), (16, 256, 1), (128, 16, 1), (16, 128, 1)):
            for f16 in (0, 1):
                assert lib.fpd_conv2d_tc_h_supported(cin, cout, k, hw, hw, f16) == 1, (cin, cout, k, hw, f16)
    assert lib.fpd_conv2d_tc_h_supported(32, 32, 3, 128, 128, 1) == 1          # stem bottleneck at 128x128
    assert lib.fpd_conv2d_tc_h_supported(160, 32, 1, 128, 128, 1) == 1         # 7x7 stem as im2col (K padded to 160)
    assert lib.fpd_conv2d_tc_h_supported(64, 64, 3, 64, 48, 1) == 1            # HRNet resolution
    assert lib.fpd_conv2d_tc_h_supported(3, 32, 7, 256, 256, 0) == 0           # raw 7x7 stem: not a tensor-core shape
    assert lib.fpd_conv2d_tc_h_supported(64, 64, 5, 64, 64, 0) == 0
    assert lib.fpd_conv2d_tc_h_supported(6, 64, 1, 64, 64, 1) == 0             # fp16 rows need Cin % 8 == 0 ...
    assert lib.fpd_conv2d_tc_h_supported(12, 64, 1, 64, 64, 0) == 1            # ... tf32 rows Cin % 4 == 0
    assert lib.fpd_conv2d_tc_h_supported(64, 24, 1, 64, 64, 0) == 0            # Cout % 16
    # pose_resnet-50/101/152 (layer2..4, the deconv head as 3x3 convs to 4 x 256 channels, and their data gradients) at
    # 256x256 and 256x192 inputs: up to 2048 channels in, 2048 out (BN-parameter shared memory is sized per launch)
    for (h, w) in ((8, 8), (8, 6), (16, 16), (16, 12), (32, 24)):
        for (cin, cout, k) in ((2048, 512, 1), (512, 2048, 1), (1024, 2048, 1), (512, 512, 3), (2048, 1024, 3),
                               (1024, 2048, 3), (1024, 256, 1), (256, 1024, 3)):
            for f16 in (0, 1):
                assert lib.fpd_conv2d_tc_h_supported(cin, cout, k, h, w, f16) == 1, (cin, cout, k, h, w, f16)
    assert lib.fpd_conv2d_tc_h_supported(4096, 512, 1, 8, 8, 1) == 0
    assert lib.fpd_conv2d_tc_h_supported(512, 4096, 1, 8, 8, 1) == 0
    # ... their weight gradients go per (Cin, Cout) chunk through the tensor-core kernels
    from fpd_b200 import ops
    assert ops.wgrad_channel_chunks(64, 64, 3) == (64, 64)                     # one launch
    assert ops.wgrad_channel_chunks(256, 256, 3) == (128, 256)                 # HRNet / ResNet layer3: Cin in two halves
    assert ops.wgrad_channel_chunks(512, 512, 3) == (128, 256)
    assert ops.wgrad_channel_chunks(2048, 1024, 3) == (128, 256)               # first deconv of ResNet-50 as a 3x3 conv
    assert ops.wgrad_channel_chunks(2048, 512, 1) == (256, 512)                # 1x1: any Cout, Cin <= 256 per launch
    assert ops.wgrad_channel_chunks(256, 1024, 1) == (256, 1024)
    assert ops.wgrad_channel_chunks(32, 17, 3) is None                         # 17-joint head: CUDA-core path
    # 3x3 weight gradients: every shape the dispatcher sends to the tensor cores (3x3, Cin in {32, 64, 128}, Cout % 32 == 0
    # up to 256), at any image size; other shapes do not
    for hw in (64, 32, 16, 8, 4):
        assert lib.fpd_conv2d_wgrad_tc3_supported(hw, hw, 64, 64, 3) == 1
    assert lib.fpd_conv2d_wgrad_tc3_supported(64, 48, 64, 32, 3) == 1
    assert lib.fpd_conv2d_wgrad_tc3_supported(64, 64, 32, 32, 3) == 1
    assert lib.fpd_conv2d_wgrad_tc3_supported(64, 64, 32, 128, 3) == 1
    assert lib.fpd_conv2d_wgrad_tc3_supported(32, 32, 128, 128, 3) == 1
    assert lib.fpd_conv2d_wgrad_tc3_supported(64, 64, 16, 32, 3) == 0          # Cin must be 32, 64 or 128
    assert lib.fpd_conv2d_wgrad_tc3_supported(64, 64, 64, 48, 3) == 0          # Cout % 32
    assert lib.fpd_conv2d_wgrad_tc3_supported(64, 64, 64, 64, 1) == 0          # 1x1: not a 3x3 shape
    # workspace of the dispatching entry point covers whichever kernel runs
    assert lib.fpd_conv2d_wgrad_tc_workspace_bytes(32, 64, 64, 64, 64, 3) >= 9 * 64 * 64 * 4


def test_bench_reference_arm_contract_on_cpu(capsys):
    """`bench.py --impl reference` (the reference's own modules from oracle/_ref on the host cores; oracle port when that
    directory is absent) prints one JSON line with the contract's keys for every config; runs here without a GPU (one
    short timed step at a reduced batch)."""
    import json
    import sys
    import types
    sys.path.insert(0, ROOT)
    import bench
    from oracle import ref_modules as R
    os.environ["FPD_CPU_THREADS"] = str(min(8, len(os.sched_getaffinity(0))))
    try:
        for name, B in (("hg_mse_s1", 2), ("hg_fpd", 1), ("hg_infer", 1)) + ((("hrnet_fpd", 1),) if R.available() else ()):
            bench.run_reference(types.SimpleNamespace(steps=1, warmup=0, gpus=1, config=name, batch=B), rank=0)
            line = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
            assert line["impl"] == "reference" and line["metric"] == "images/sec" and line["unit"] == "images/s"
            assert line["value"] > 0 and line["higher_is_better"] is True and line["n_gpus"] == 1
            assert line["steps"] == 1 and line["warmup"] == 0
            assert line["config"] == bench.workload_config(name, 1, bench.CONFIGS[name]["batch"])   # = the GPU arm's config
            assert line["cpu_baseline"]["kind"] == ("reference" if R.available() else "port")
            assert line["cpu_baseline"]["cores"] >= 1
            assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["d2h_bytes_per_step"] == 0
    finally:
        os.environ.pop("FPD_CPU_THREADS", None)
    # other ranks of a torchrun launch stay silent
    bench.run_reference(types.SimpleNamespace(steps=1, warmup=0, gpus=2, config="hg_fpd", batch=1), rank=1)
    assert capsys.readouterr().out == ""
