"""Flip-test inference as one replayable CUDA graph (BASELINE configs[4]).

What the reference does per validation batch (lib/core/function.py:212-240, lib/core/inference.py:18-46): forward,
`np.flip(input.cpu().numpy(), 3)` + H2D, second forward, D2H of the flipped heat-maps, `flip_back` in numpy, H2D, shift by
one pixel, average, D2H of the merged heat-maps, numpy arg-max. Here, per batch:

    graph replay { image -> NHWC and W-mirrored NHWC (one pass each)
                   forward (eval BN, cached 3xFP16 weights)      | second stream: forward of the mirrored image
                   fused flip_back + shift + average + arg-max -> idx[B,J], maxval[B,J] (+ merged heat-maps)
                   [optional box NMS of the detector boxes that produced the crops: lib/nms, csrc/nms.cu]
                   [decode=True: merged map -> NCHW -> JointsMSELoss, JointsOHKMMSELoss or JointsKLDLoss (loss3), get_final_preds
                    (preds; DARK's decode with post_process="dark"), accuracy() counts (pck), all on the device,
                    bit-identical to lib/core/function.py's eager route] }

Only [B,J] indices and maxima (or [B,J,3] predictions, 3 loss floats and [J,2] counts) need to cross PCIe. The module must be one of fpd_b200.lib.models (hourglass / pose_hrnet).
"""
import torch

from . import ops


def _post_process(post_process):
    """The decode a post_process argument selects: "dark", or a bool (the quarter-pixel nudge or none)."""
    if isinstance(post_process, str):
        if post_process != "dark":
            raise ValueError("post_process must be a bool or 'dark', got %r" % (post_process,))
        return post_process
    return bool(post_process)


def _temperature(topk, temperature):
    """The decode stage's JointsKLDLoss temperature: 0 (another criterion) or finite and > 0, never with a topk."""
    t = ops._check_temperature(temperature, "temperature", True)
    if t and topk:
        raise ValueError("the criterion is JointsOHKMMSELoss (topk) or JointsKLDLoss (temperature), not both")
    return t


class FlipTestInference:
    def __init__(self, net, flip_pairs, shift_heatmap=True, flip_test=True, use_graph=True, want_avg=True, decode=False):
        """decode: also run validation's loss, keypoint decode and PCK counts in the graph; __call__ then needs inv,
        target and target_weight."""
        self.net = net
        self.flip_test = flip_test
        self.shift = bool(shift_heatmap)
        self.use_graph = use_graph
        self.decode = decode
        self.want_avg = want_avg or decode
        self.static_extra = None
        self.pairs = [tuple(p) for p in flip_pairs]
        self.graph = None
        self.static_x = None
        self.static_boxes = None
        self.result = None
        self._shape = None
        self._gen = -1
        self._side = torch.cuda.Stream() if flip_test else None
        self._keep = None
        self.nms_thresh = None
        self._stage_x = self._copy_stream = self._stage_ev = self._stage_free = None
        self._staged_for = None
        net.eval()

    def _perm(self, J, device):
        p = list(range(J))
        for a, b in self.pairs:
            p[a], p[b] = b, a
        return torch.tensor(p, dtype=torch.int32, device=device)

    def _body(self, x, boxes, extra=None):
        eng = self.net.engine()
        main = torch.cuda.current_stream()
        nhwc = ops.nchw_to_nhwc(x)
        ctx_f = None
        if self.flip_test:
            self._side.wait_stream(main)
            with torch.cuda.stream(self._side):
                nhwc_f = ops.nchw_to_nhwc_flipw(x)
                ctx_f = eng.forward(x, False, record_tape=False, shared_stem={"img": x, "nhwc": nhwc_f})
        ctx = eng.forward(x, False, record_tape=False, shared_stem={"img": x, "nhwc": nhwc})
        hm = ctx.outs[-1].data
        hm_f = None
        if ctx_f is not None:
            main.wait_stream(self._side)
            hm_f = ctx_f.outs[-1].data
        J = hm.shape[-1]
        if getattr(self, "_perm_t", None) is None or self._perm_t.numel() != J:
            self._perm_t = self._perm(J, x.device)
        avg, idx, maxval = ops.flip_merge_argmax(hm, hm_f, self._perm_t if hm_f is not None else None, shift=self.shift,
                                                 want_avg=self.want_avg)
        keep = num = None
        if boxes is not None:
            keep, num = ops.nms_device(boxes, self.nms_thresh)
        res = {"idx": idx, "maxval": maxval, "avg_nhwc": avg, "nms_keep": keep, "nms_num": num}
        out_nchw = None
        if self.decode:
            # the loss validate() computes: the criterion on the NCHW merged map (same kernel, same summation order)
            out_nchw = ops.nhwc_to_nchw(avg)
            B, J = idx.shape
            tw = extra["target_weight"].reshape(B, J) if extra["use_target_weight"] else None
            if extra["temperature"]:
                res["loss3"], _ = ops.joints_kld(out_nchw, extra["target"], tw, extra["temperature"], want_grad=False)
            elif extra["topk"]:
                res["loss3"], _ = ops.joints_ohkm_mse(out_nchw, extra["target"], tw, extra["topk"], want_grad=False)
            else:
                res["loss3"], _ = ops.joints_mse(out_nchw, extra["target"], tw, want_grad=False)
            if extra["post_process"] == "dark":
                res["preds"] = ops.final_preds_dark(avg, idx, maxval, extra["inv"], extra["blur_kernel"])
            else:
                res["preds"] = ops.final_preds(avg, idx, maxval, extra["inv"], extra["post_process"])
            res["pck"], _ = ops.pck_counts(idx, maxval, extra["target"])
        self._keep = (ctx, ctx_f, nhwc, out_nchw)      # every intermediate stays referenced: the graph pool never recycles them
        return res

    def _extra(self, inv, target, target_weight, use_target_weight, post_process, topk, blur_kernel, temperature,
               static):
        """The decode stage's inputs on the device: fresh copies, or refills of the graph's static buffers."""
        if not self.decode:
            return None
        if inv is None or target is None or target_weight is None:
            raise ValueError("FlipTestInference(decode=True) needs inv, target and target_weight")
        inv = torch.as_tensor(inv, dtype=torch.float64)
        if static is None:
            dev = torch.device("cuda", torch.cuda.current_device())

            def own(t, dtype):          # always a new buffer: a graph must not alias the caller's tensors
                return torch.empty(tuple(t.shape), dtype=dtype, device=dev).copy_(t)
            return {"inv": own(inv, torch.float64), "target": own(target, torch.float32),
                    "target_weight": own(target_weight, torch.float32),
                    "use_target_weight": bool(use_target_weight), "post_process": _post_process(post_process),
                    "topk": int(topk), "blur_kernel": int(blur_kernel),
                    "temperature": _temperature(topk, temperature)}
        static["inv"].copy_(inv, non_blocking=True)
        static["target"].copy_(target, non_blocking=True)
        static["target_weight"].copy_(target_weight, non_blocking=True)
        return static

    def _stage(self, x):
        main = torch.cuda.current_stream()
        if self._staged_for is not None and self._staged_for is x:
            main.wait_event(self._stage_ev)
            self.static_x.copy_(self._stage_x, non_blocking=True)
            self._stage_free.record(main)
        else:
            self.static_x.copy_(x, non_blocking=True)
        self._staged_for = None

    def _prefetch(self, next_x):
        """H2D of the next batch (pinned host tensor) on a copy stream, under this batch's graph replay."""
        if next_x is None or next_x.is_cuda or not next_x.is_pinned() or tuple(next_x.shape) != tuple(self.static_x.shape):
            return
        if self._stage_x is None or self._stage_x.shape != self.static_x.shape:
            self._stage_x = torch.empty_like(self.static_x)
            self._copy_stream = torch.cuda.Stream()
            self._stage_ev, self._stage_free = torch.cuda.Event(), torch.cuda.Event()
            self._stage_free.record(torch.cuda.current_stream())
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._stage_free)
            self._stage_x.copy_(next_x, non_blocking=True)
            self._stage_ev.record(self._copy_stream)
        self._staged_for = next_x

    def __call__(self, x, boxes_sorted=None, nms_thresh=0.6, next_x=None, inv=None, target=None, target_weight=None,
                 use_target_weight=True, post_process=True, topk=0, blur_kernel=11, temperature=0.0):
        """x: [B,3,H,W] fp32, CUDA or pinned host. boxes_sorted: optional device [n,5] detector boxes sorted by score.
        next_x: optional pinned host tensor = the NEXT batch (its H2D copy overlaps this batch; pass it as `x` next time).
        With decode=True: inv host float64 [B,6] heat-map -> image matrices (lib.core.inference.inverse_affines of the
        batch's centres / scales), target [B,J,h,w] and target_weight [B,J,1] (host or device), use_target_weight (the
        criterion's), post_process (config.TEST.POST_PROCESS; "dark" decodes with ops.final_preds_dark and a
        blur_kernel-tap blur instead of the quarter-pixel nudge), topk (the JointsOHKMMSELoss criterion's topk; 0 for
        JointsMSELoss) and temperature (the JointsKLDLoss criterion's temperature; 0 for the other two).
        Returns a dict of DEVICE tensors (static across calls in graph mode): idx int32 [B,J] (flat arg-max, first maximum),
        maxval [B,J], avg_nhwc [B,h,w,J] merged heat-maps, nms_keep / nms_num; with decode=True also preds [B,J,3]
        (get_final_preds: x, y, maxval), loss3 [3] (loss3[0] = the criterion's value) and pck int32 [J,2] (per joint:
        valid, hit; lib.core.evaluate.pck_from_counts gives accuracy()'s acc / avg_acc / cnt)."""
        self.net.engine().check_input_size(*x.shape[2:])     # before any copy, launch or capture
        self.nms_thresh = float(nms_thresh)
        if not self.use_graph:
            xd = x.cuda(non_blocking=True).float().contiguous()
            return self._body(xd, boxes_sorted, self._extra(inv, target, target_weight, use_target_weight, post_process,
                                                            topk, blur_kernel, temperature, None))
        shape = (tuple(x.shape), None if boxes_sorted is None else tuple(boxes_sorted.shape), self.nms_thresh)
        if self.decode:
            shape += (tuple(target.shape), tuple(target_weight.shape), bool(use_target_weight),
                      _post_process(post_process), int(topk), int(blur_kernel), _temperature(topk, temperature))
        gen = self.net.engine().generation
        if self.graph is None or shape != self._shape or gen != self._gen:
            xd = x.cuda(non_blocking=True).float().contiguous()
            self.static_x = torch.empty_like(xd)
            self.static_x.copy_(xd)
            self.static_boxes = None if boxes_sorted is None else boxes_sorted.clone()
            self.static_extra = self._extra(inv, target, target_weight, use_target_weight, post_process, topk, blur_kernel,
                                            temperature, None)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                with torch.no_grad():
                    self._body(self.static_x, self.static_boxes, self.static_extra)      # warm-up: lazy init, workspaces, weight cache
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            from . import _native as N
            n0 = N.lib().fpd_launch_count()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self.result = self._body(self.static_x, self.static_boxes, self.static_extra)
            self.launches = int(N.lib().fpd_launch_count() - n0)
            self._shape, self._gen = shape, self.net.engine().generation
        self._stage(x)
        if boxes_sorted is not None:
            self.static_boxes.copy_(boxes_sorted, non_blocking=True)
        self._extra(inv, target, target_weight, use_target_weight, post_process, topk, blur_kernel, temperature,
                    self.static_extra)
        self.graph.replay()
        self._prefetch(next_x)
        return self.result
