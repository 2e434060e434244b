"""What detect.py --multi-scale costs for a batch of 32 HRSC-like 1024x768 sources at the two sizes drawn for a base
size of 608 (multiscale_sizes(608) under numpy seed 0), through the Darknet-53 yolov3 graph with random weights, one
class, conf 0.5, NMS 0.5, at most 20 000 candidates per image and size:

  (a) nms.detect_multiscale on the whole batch: device time from CUDA events around the call, and the host clock
      ending in a device synchronise; per stage, the kernel time of one separate call under torch.profiler (uploads and
      letterbox, forwards, per-size detection, merge, second detection);
  (b) multi_detect's loop restated per image at batch 1 (one upload per image, then per size letterbox, forward,
      detect_postprocess_classes with one host read of the kept count, scale_coords and round; then the cross-scale
      detection): host clock ending in a device synchronise.

The two paths alternate in one process, and their detections are checked to be equal before anything is reported.
With random weights about half of the 545 832 rows per image pass the threshold, so the two NMS stages dominate (as in
bench.py's detect line).  The card's name, power limit and SM clock are read in the same run.

    python tools/multiscale_detect_times.py OUT_DIR [--reps 3]

Writes OUT_DIR/multiscale_detect_times.json.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))

BATCH, SRC_HW, BASE, CONF, NMS, CAP = 32, (768, 1024), 608, 0.5, 0.5, 20000


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        name, pl, mx, sm = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit_w": float(pl), "sm_max_mhz": float(mx), "sm_mhz": float(sm)}
    except Exception as e:  # noqa: BLE001 -- report, do not fail the measurement
        return {"error": repr(e)[:200]}


def make_model():
    import helpers
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    m = pkg.Darknet(cfgs.yolov3_cfg(classes=1), {"context_factor": 1.0}, arc="default")
    helpers.init_darknet_weights(m, seed=5)
    return m.cuda().eval()


def make_images():
    g = np.random.RandomState(1)
    return [g.randint(0, 256, SRC_HW + (3,)).astype(np.uint8) for _ in range(BATCH)]


def batched(model, images, sizes):
    import torch
    from rotate_yolov3_b200 import detect_multiscale
    from rotate_yolov3_b200.nms import detections_per_image
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    res = detect_multiscale(model, images, sizes, CONF, NMS, CAP)
    e1.record()
    torch.cuda.synchronize()
    host_ms = (time.perf_counter() - t0) * 1e3
    return detections_per_image(res), e0.elapsed_time(e1), host_ms


def per_image(model, images, sizes):
    """multi_detect (detect.py:76-101) with the package's per-image pieces, batch 1"""
    import torch
    from rotate_yolov3_b200 import letterbox, scale_coords
    from rotate_yolov3_b200.nms import detect_postprocess_classes, detections_per_image
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = []
    with torch.no_grad():
        for img0 in images:
            src = torch.from_numpy(img0).pin_memory().cuda(non_blocking=True)
            all_pre = []
            for s in sizes:
                img, _ = letterbox([src], s)
                io, _ = model(img)
                r = detect_postprocess_classes(io, CONF, 0.95, CAP)
                k = int(r["num_keep"][0])
                if k:
                    det = r["dets"][0][r["keep"][0, :k]]
                    det[:, :4] = scale_coords((s, s), det[:, :4], img0.shape).round()
                    all_pre.append(det)
            if not all_pre:
                out.append(None)
                continue
            merged = torch.cat(all_pre, 0)
            out.append(detections_per_image(detect_postprocess_classes(merged[None].contiguous(), CONF, NMS,
                                                                       len(merged)))[0])
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def stage_times(model, images, sizes):
    """kernel and copy time of one batched call by stage, from the profiler's device events"""
    import torch
    from rotate_yolov3_b200 import detect_multiscale
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        detect_multiscale(model, images, sizes, CONF, NMS, CAP)
        torch.cuda.synchronize()
    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                 key=lambda e: e.time_range.start)
    merge = [i for i, e in enumerate(evs) if "merge_scales" in e.name]
    assert len(merge) == 1, [e.name for e in evs][:50]
    stages = {"upload_and_letterbox": 0.0, "forwards": 0.0, "per_size_detection": 0.0, "merge": 0.0,
              "second_detection": 0.0}
    for i, e in enumerate(evs):
        n, us = e.name, e.time_range.elapsed_us()
        if i == merge[0]:
            stages["merge"] += us
        elif i > merge[0]:
            stages["second_detection"] += us
        elif "letterbox" in n or "Memcpy" in n:
            stages["upload_and_letterbox"] += us
        elif any(k in n for k in ("sel_", "rnms", "cub", "Radix", "Sort")):
            stages["per_size_detection"] += us
        else:
            stages["forwards"] += us
    return {k: v / 1e3 for k, v in stages.items()}


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("out_dir")
    ap_.add_argument("--reps", type=int, default=3)
    args = ap_.parse_args()
    import torch
    from rotate_yolov3_b200 import multiscale_sizes
    sizes = multiscale_sizes(BASE, np.random.RandomState(0))
    model = make_model()
    images = make_images()
    got, _, _ = batched(model, images, sizes)                      # warm-up: plans of both sizes, module loads
    want, _ = per_image(model, images, sizes)
    runs = []
    for _ in range(args.reps):
        got, dev_ms, host_ms = batched(model, images, sizes)
        want, loop_ms = per_image(model, images, sizes)
        runs.append({"batched_device_ms": dev_ms, "batched_host_ms": host_ms, "per_image_host_ms": loop_ms})
    for b, (g, w) in enumerate(zip(got, want)):
        assert (g is None) == (w is None), b
        assert g is None or (g.shape == w.shape and torch.equal(g, w)), (b, None if g is None else g.shape, w.shape)
    stages = stage_times(model, images, sizes)
    med = lambda k: float(np.median([r[k] for r in runs]))
    result = {
        "gpu": gpu_info(), "torch": torch.__version__, "batch": BATCH, "source_hw": SRC_HW, "sizes": sizes,
        "conf_thres": CONF, "nms_thres": NMS, "cap": CAP,
        "kept": [0 if g is None else len(g) for g in got],
        "batched_device_ms": med("batched_device_ms"), "batched_host_ms": med("batched_host_ms"),
        "per_image_host_ms": med("per_image_host_ms"), "batched_stage_kernel_ms": stages, "runs": runs,
    }
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "multiscale_detect_times.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
