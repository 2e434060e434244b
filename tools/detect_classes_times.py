"""What class-aware post-processing costs at the bench's detect shape: a random-init yolov3 with nc classes on 32 images
of 608x608, conf 0.5, NMS 0.5, at most 20 000 candidates per image, for nc in {1, 3, 15}:

  (a) nms.detect_postprocess_classes: device-side selection + one class-aware segmented NMS, no host sync;
  (b) the per-image per-class host loop available without it: nms_filter -> stable top-cap -> r_nms per class;
  (c) at nc = 1, nms.detect_postprocess (class-agnostic).

Each is timed with CUDA events after a warm-up call; then, in a separate torch.profiler run, the device time of
rnms_mask_kernel per call of (a) (of (c) at nc = 1).  The card's name, power limit and SM clock are read in the same run.

    python tools/detect_classes_times.py OUT_DIR [--tree DIR] [--iters 10] [--loop-iters 2]

--tree imports rotate_yolov3_b200 from another checkout (for example an earlier commit, built in place), so that two
versions can be measured in one session; (a) is skipped when that package does not have it.  Writes
OUT_DIR/detect_classes_times.json.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "tests"))

BATCH, CONF, THR, CAP = 32, 0.5, 0.5, 20000


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        name, pl, mx, sm = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit_w": float(pl), "sm_max_mhz": float(mx), "sm_mhz": float(sm)}
    except Exception as e:  # noqa: BLE001 -- report, do not fail the measurement
        return {"error": repr(e)[:200]}


def event_ms(fn, iters):
    import torch
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def mask_kernel_ms(fn, calls):
    """device time of rnms_mask_kernel per call of fn, from a torch.profiler trace of `calls` calls"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    total_us, launches = 0.0, 0
    for ev in prof.key_averages():
        if "rnms_mask_kernel" in ev.key:
            total_us += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            launches += ev.count
    return total_us / 1000.0 / calls, launches // calls


def bench_io(nc):
    import torch
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    from helpers import init_darknet_weights
    model = pkg.Darknet(cfgs.yolov3_cfg(classes=nc), {"context_factor": 1.0}, arc="default")
    init_darknet_weights(model, seed=1)
    model = model.cuda().eval()
    x = torch.rand(BATCH, 3, 608, 608, generator=torch.Generator().manual_seed(0)).cuda()
    with torch.no_grad():
        io, _ = model(x)
    del model, x
    torch.cuda.empty_cache()
    return io


def host_loop(io):
    """today's multi-class route at a cap: per image nms_filter -> stable top-cap -> input order -> r_nms per class"""
    import torch
    from rotate_yolov3_b200.nms import nms_filter, r_nms
    out = []
    for b in range(io.shape[0]):
        cand = nms_filter(io[b].clone(), CONF, 2.0)
        top = torch.sort(torch.argsort(cand[:, 5], descending=True, stable=True)[:CAP]).values
        sel = cand[top]
        keep = []
        for c in sel[:, 7].unique():
            idx = torch.nonzero(sel[:, 7] == c).flatten()
            keep.append(idx[r_nms(sel[idx, :6].contiguous(), THR)])
        out.append(sel[torch.sort(torch.cat(keep)).values] if keep else sel[:0])
    torch.cuda.synchronize()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--tree", default=REPO, help="checkout whose rotate_yolov3_b200 is measured")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--loop-iters", type=int, default=2)
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.tree))
    import torch
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import nms
    os.makedirs(a.out, exist_ok=True)
    res = {"gpu": gpu_info(), "tree": os.path.abspath(a.tree), "lib": pkg._lib.LIB_PATH, "batch": BATCH, "cap": CAP,
           "conf_thres": CONF, "nms_thres": THR, "rows": []}
    print(json.dumps(res["gpu"]), flush=True)
    has_classes = hasattr(nms, "detect_postprocess_classes")
    for nc in (1, 3, 15):
        io = bench_io(nc)
        row = {"nc": nc}
        fa = (lambda: nms.detect_postprocess_classes(io, CONF, THR, CAP)) if has_classes else None
        fc = (lambda: nms.detect_postprocess(io, CONF, THR, CAP)) if nc == 1 else None
        if fa:
            r = fa()
            row["candidates"] = int(r["counts"].sum())
            row["kept"] = int(r["num_keep"].sum())
            row["a_classes_ms"] = event_ms(fa, a.iters)
        row["b_host_loop_ms"] = event_ms(lambda: host_loop(io), a.loop_iters)
        if fc:
            row["c_agnostic_ms"] = event_ms(fc, a.iters)
        if fa:
            row["a_mask_kernel_ms"], row["a_mask_launches"] = mask_kernel_ms(fa, 3)
        if fc:
            row["c_mask_kernel_ms"], row["c_mask_launches"] = mask_kernel_ms(fc, 3)
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
        del io
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "detect_classes_times.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"gpu": res["gpu"], "gpu_after": res["gpu_after"], "lib": res["lib"]}), flush=True)


if __name__ == "__main__":
    main()
