"""Error report for the network-level parity on a GPU host: per-stack relative error of the CUDA path vs the
oracle (fp32 and fp64), plus the oracle-fp32-vs-fp64 noise floor, for several configs / precision modes."""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NS = types.SimpleNamespace


def rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


def main():
    import fpd_b200  # noqa: F401
    from fpd_b200.lib.models import hourglass as H
    from oracle import hourglass_oracle as O
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    for (f, s, B, hw, training) in [(64, 2, 2, 64, True), (128, 4, 4, 256, True), (128, 4, 32, 256, True),
                                    (256, 8, 4, 256, False)]:
        torch.manual_seed(0)
        cfg = NS(MODEL=NS(EXTRA=NS(NUM_FEATURES=f, NUM_STACKS=s, NUM_BLOCKS=1), NUM_JOINTS=16))
        net = H.get_pose_net(cfg, True).cuda()
        net.train(training)
        x = torch.randn(B, 3, hw, hw, device="cuda")
        sd = {k: v.clone() for k, v in net.state_dict().items()}
        sd64 = {k: (v.double() if v.is_floating_point() else v.clone()) for k, v in sd.items()}
        with torch.no_grad():
            ref32 = O.hourglass_net({k: v.clone() for k, v in sd.items()}, x, s, training=training)
            ref64 = O.hourglass_net(sd64, x.double(), s, training=training)
            for mode in ("tf32x3", "tf32"):
                os.environ["FPD_PRECISION"] = mode
                net.load_state_dict(sd)
                got = net(x)
                print("cfg f=%d s=%d B=%d hw=%d train=%s mode=%-6s vs_fp32 %s  vs_fp64 %s" % (
                    f, s, B, hw, training, mode, ["%.2e" % rel(a, b) for a, b in zip(got, ref32)],
                    ["%.2e" % rel(a, b) for a, b in zip(got, ref64)]), flush=True)
            print("   torch fp32 vs fp64 noise floor        %s" % ["%.2e" % rel(a, b) for a, b in zip(ref32, ref64)],
                  flush=True)
        del os.environ["FPD_PRECISION"]


if __name__ == "__main__":
    main()
