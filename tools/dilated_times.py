"""What the multi-branch dilated graph costs in eval: the forward of cfg/yolov3-m.cfg (16 heads, 36 dilated convs run as
phase-decomposed ordinary convs) against cfg/yolov3.cfg at the same batch and image size (416 and 512), alternated
three times, CUDA graphs on; the share of the yolov3-m forward taken by the phase passes (ryolo_dilate_split / _merge
launches of the plan replayed on their own); and each phase kernel at the 416 shapes against a device-to-device copy of
the same bytes.  CUDA events throughout; the card's name, power limit and SM clock are read in the same run.

    python tools/dilated_times.py OUT_DIR [--batch 16] [--iters 20] [--train-batch 8]

The training step of both graphs is timed too (fixed head cotangent in place of the loss).

Writes OUT_DIR/dilated_times.json.  Needs a GPU."""
import argparse
import ctypes
import gc
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "tools"))

from se_step_times import event_ms, gpu_info  # noqa: E402


def _model(cfg):
    import rotate_yolov3_b200 as pkg
    from helpers import init_darknet_weights
    from builders import m_cfg_text
    text = m_cfg_text(cfg)
    m = pkg.Darknet(text, {"context_factor": 1.0}, arc="default")
    return init_darknet_weights(m, seed=1).cuda().eval()


def _phase_steps(m, x):
    """the plan's split / merge launches only, in plan order"""
    from rotate_yolov3_b200 import _lib
    lib, st, b = _lib.lib, _lib.stream_ptr(x.device), x.shape[0]
    steps = [(k, a) for k, a in m._plan["steps"] if k in ("dsplit", "dmerge")]

    def run():
        for k, a in steps:
            if k == "dsplit":
                lib.ryolo_dilate_split(ctypes.c_void_p(a["x"]), a["xcs"], b, a["h"], a["w"], a["c"], a["dh"], a["dw"],
                                       _lib.ptr(a["xp"]), a["xp"].shape[-1], st)
            else:
                lib.ryolo_dilate_merge(_lib.ptr(a["yp"]), a["yp"].shape[-1], b, a["h"], a["w"], a["c"], a["dh"], a["dw"],
                                       ctypes.c_void_p(a["r"]) if a["r"] else None, a["rcs"], 0, ctypes.c_void_p(a["y"]),
                                       a["ycs"], st)
    return run, steps


def forward_times(batch, size, iters):
    import torch
    out = {}
    models = {c: _model(c) for c in ("cfg/yolov3.cfg", "cfg/yolov3-m.cfg")}
    x = torch.rand(batch, 3, size, size, device="cuda")
    for m in models.values():
        m.use_cuda_graph = True
        with torch.no_grad():
            m(x)
    for rep in range(3):
        for c, m in models.items():
            with torch.no_grad():
                out.setdefault(c, []).append(event_ms(lambda: m(x), iters))
    m = models["cfg/yolov3-m.cfg"]
    run, steps = _phase_steps(m, x)
    phase_ms = event_ms(run, iters)
    res = {"batch": batch, "size": size, "eval_ms": {c: min(v) for c, v in out.items()}, "eval_ms_runs": out,
           "phase_ms": phase_ms, "phase_launches": len(steps),
           "phase_share": phase_ms / min(out["cfg/yolov3-m.cfg"])}
    del models, m
    gc.collect()
    torch.cuda.empty_cache()
    return res


def train_times(batch, size, iters):
    """training step (forward with batch-statistics BN, backward of sum(p * G) with a fixed cotangent G in place of the
    loss), CUDA graphs on, both graphs alternated three times"""
    import torch
    out = {}
    models = {c: _model(c).train() for c in ("cfg/yolov3.cfg", "cfg/yolov3-m.cfg")}
    x = torch.rand(batch, 3, size, size, device="cuda")
    steps = {}
    for c, m in models.items():
        m.use_cuda_graph = True
        gs = [torch.randn_like(p) for p in m(x)]
        m.zero_grad(set_to_none=True)

        def step(m=m, gs=gs):
            ps = m(x)
            sum((p * g).sum() for p, g in zip(ps, gs)).backward()
        steps[c] = step
        step()
    for rep in range(3):
        for c in models:
            out.setdefault(c, []).append(event_ms(steps[c], iters))
    res = {"batch": batch, "size": size, "train_ms": {c: min(v) for c, v in out.items()}, "train_ms_runs": out}
    del models, steps
    gc.collect()
    torch.cuda.empty_cache()
    return res


def kernel_bandwidth(batch, iters):
    """each (grid, channels, dilation) of yolov3-m at 416: split and merge (with residual) against a copy of the bytes the
    kernel must move (split: read H*W*C, write Hp*Wp*C*dh*dw; merge: read 2 H*W*C, write H*W*C)"""
    import torch
    from rotate_yolov3_b200 import _lib
    from rotate_yolov3_b200 import layout as L
    lib, st = _lib.lib, _lib.stream_ptr(torch.device("cuda"))
    rows = []
    for hw, c in ((13, 1024), (26, 512), (52, 256)):
        x = L.alloc_padded(batch, hw, hw, c, "cuda")
        x[:, 1:-1, 1:-1].normal_()
        r, y = torch.randn_like(x), torch.zeros_like(x)
        for dh, dw in ((1, 2), (2, 1), (1, 4), (4, 1), (1, 8), (8, 1)):
            hp, wp = -(-hw // dh), -(-hw // dw)
            xp = L.alloc_padded(batch * dh * dw, hp, wp, c, "cuda")
            t_split = event_ms(lambda: lib.ryolo_dilate_split(_lib.ptr(x), c, batch, hw, hw, c, dh, dw, _lib.ptr(xp), c,
                                                              st), iters)
            t_merge = event_ms(lambda: lib.ryolo_dilate_merge(_lib.ptr(xp), c, batch, hw, hw, c, dh, dw, _lib.ptr(r), c,
                                                              0, _lib.ptr(y), c, st), iters)
            nat = batch * hw * hw * c * 2
            ph = batch * dh * dw * hp * wp * c * 2
            src = torch.empty(nat + ph, dtype=torch.uint8, device="cuda")
            dst = torch.empty_like(src)
            t_copy_s = event_ms(lambda: dst.copy_(src), iters)
            src2 = torch.empty(3 * nat // 2, dtype=torch.uint8, device="cuda")
            dst2 = torch.empty_like(src2)
            t_copy_m = event_ms(lambda: dst2.copy_(src2), iters)
            rows.append({"grid": hw, "c": c, "dil": [dh, dw], "split_ms": t_split, "merge_ms": t_merge,
                         "split_GBps": (nat + ph) / t_split / 1e6, "merge_GBps": 3 * nat / t_merge / 1e6,
                         "copy_GBps_split_bytes": 2 * (nat + ph) / t_copy_s / 1e6,
                         "copy_GBps_merge_bytes": 3 * nat / t_copy_m / 1e6})
            del xp, src, dst, src2, dst2
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--train-batch", type=int, default=8)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    res = {"gpu": gpu_info(), "batch": a.batch}
    res["kernels_416"] = kernel_bandwidth(a.batch, 50)
    res["forward"] = [forward_times(a.batch, s, a.iters) for s in (416, 512)]
    res["train"] = [train_times(a.train_batch, s, a.iters) for s in (416, 512)]
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "dilated_times.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["gpu"]))
    for f_ in res["forward"]:
        print("eval %d^2 b%d: yolov3 %.2f ms, yolov3-m %.2f ms, phase passes %.2f ms (%.1f%%, %d launches)" % (
            f_["size"], f_["batch"], f_["eval_ms"]["cfg/yolov3.cfg"], f_["eval_ms"]["cfg/yolov3-m.cfg"], f_["phase_ms"],
            100 * f_["phase_share"], f_["phase_launches"]))
    for t in res["train"]:
        print("train %d^2 b%d: yolov3 %.2f ms, yolov3-m %.2f ms" % (
            t["size"], t["batch"], t["train_ms"]["cfg/yolov3.cfg"], t["train_ms"]["cfg/yolov3-m.cfg"]))
    for r in res["kernels_416"]:
        print("%3d^2 x %4d dil %s: split %.1f GB/s, merge %.1f GB/s, copy %.1f / %.1f GB/s" % (
            r["grid"], r["c"], r["dil"], r["split_GBps"], r["merge_GBps"], r["copy_GBps_split_bytes"],
            r["copy_GBps_merge_bytes"]))


if __name__ == "__main__":
    main()
