"""What the focal objectness costs next to the plain BCE: ryolo_obj_bce_fwd / _bwd against ryolo_obj_focal_fwd / _bwd at
the three batch-64 608 x 608 heads (NCHW [64, 72 * 7, ny, ny] buffers read as the [64, 72, ny, ny, 7] view Darknet
returns, ny = 76, 38, 19), timed with CUDA events over 50 launches, alternated three times, and set next to a
device-to-device copy that moves the same bytes in the same process.  The card's name, power limit and SM clock are read
in the same run.

    python tools/loss_kernel_times.py OUT_DIR [--iters 50] [--gamma 0.5]

Writes OUT_DIR/loss_kernel_times.json.  Needs a GPU.  Bytes per cell the kernels need: forward reads the objectness
logit and tobj (8 B); backward reads the same and writes the 7-channel cotangent (8 + 28 B)."""
import argparse
import ctypes
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from se_step_times import event_ms, gpu_info  # noqa: E402

B, NA, NO = 64, 72, 7
FWD_BYTES, BWD_BYTES = 8, 36


def head_times(ny, iters, gamma, reps=3):
    import torch
    import rotate_yolov3_b200 as pkg
    L = pkg._lib
    g = torch.Generator(device="cuda").manual_seed(ny)
    buf = torch.randn(B, NA * NO, ny, ny, generator=g, device="cuda") * 3.0
    x = buf.view(B, NA, NO, ny, ny).permute(0, 1, 3, 4, 2)
    tobj = (torch.rand(B, NA, ny, ny, generator=g, device="cuda") < 0.01).float()
    grad = torch.empty_strided(x.shape, x.stride(), dtype=torch.float32, device="cuda")
    s = torch.zeros(1, dtype=torch.float64, device="cuda")
    scale = torch.full((1,), 1e-6, device="cuda")
    strides = (ctypes.c_longlong * 5)(*x.stride())
    st = L.stream_ptr()
    args = (L.ptr(x), strides, B, NA, ny, ny, NO, 5, L.ptr(tobj), 1.0)
    fns = {
        "bce_fwd": lambda: L.check(L.lib.ryolo_obj_bce_fwd(*args, L.ptr(s), st), "bce_fwd"),
        "focal_fwd": lambda: L.check(L.lib.ryolo_obj_focal_fwd(*args, gamma, L.ptr(s), st), "focal_fwd"),
        "bce_bwd": lambda: L.check(L.lib.ryolo_obj_bce_bwd(*args, L.ptr(scale), L.ptr(grad), st), "bce_bwd"),
        "focal_bwd": lambda: L.check(L.lib.ryolo_obj_focal_bwd(*args, gamma, L.ptr(scale), L.ptr(grad), st), "focal_bwd"),
    }
    cells = B * NA * ny * ny
    # a copy of n bytes reads n and writes n: copies of FWD_BYTES / 2 and BWD_BYTES / 2 bytes per cell move what the
    # kernels move
    src_f, src_b = torch.empty(cells * FWD_BYTES // 8, device="cuda"), torch.empty(cells * BWD_BYTES // 8, device="cuda")
    dst_f, dst_b = torch.empty_like(src_f), torch.empty_like(src_b)
    copies = {"copy_fwd": lambda: dst_f.copy_(src_f), "copy_bwd": lambda: dst_b.copy_(src_b)}
    runs = []
    for _ in range(reps):
        r = {k: event_ms(f, iters) for k, f in copies.items()}
        for k in ("bce_fwd", "focal_fwd", "bce_bwd", "focal_bwd"):
            r[k] = event_ms(fns[k], iters)
        runs.append(r)
    best = {k: min(r[k] for r in runs) for k in runs[0]}
    row = {"head": "%d^2" % ny, "cells": cells, "runs_ms": runs}
    for k, t in best.items():
        nbytes = cells * (FWD_BYTES if k.endswith("fwd") else BWD_BYTES)
        row[k + "_ms"] = t
        row[k + "_gbps"] = nbytes / t / 1e6
    row["focal_over_bce_fwd"] = best["focal_fwd"] / best["bce_fwd"]
    row["focal_over_bce_bwd"] = best["focal_bwd"] / best["bce_bwd"]
    del buf, x, grad, src_f, src_b, dst_f, dst_b
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--gamma", type=float, default=0.5)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "loss_kernel_times needs a GPU"
    os.makedirs(a.out, exist_ok=True)
    res = {"gpu": gpu_info(), "gamma": a.gamma, "iters": a.iters, "heads": []}
    print(json.dumps(res["gpu"]), flush=True)
    for ny in (76, 38, 19):
        row = head_times(ny, a.iters, a.gamma)
        res["heads"].append(row)
        print(json.dumps({k: v for k, v in row.items() if k != "runs_ms"}), flush=True)
    tot = {k: sum(r[k + "_ms"] for r in res["heads"]) for k in ("bce_fwd", "focal_fwd", "bce_bwd", "focal_bwd",
                                                                 "copy_fwd", "copy_bwd")}
    res["total_ms"] = tot
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "loss_kernel_times.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"total_ms": tot, "gpu_after": res["gpu_after"]}), flush=True)


if __name__ == "__main__":
    main()
