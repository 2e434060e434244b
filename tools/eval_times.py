"""What the mAP evaluation costs over a pass the size of HRSC2016's test split (444 images) at batch 16, 512x512,
conf 0.001 (test.py's), NMS 0.5, at most 20 000 candidates per image, one class:

  (a) metrics.Evaluator: add() per batch, timed with CUDA events over the whole pass, and compute(), timed on the host
      clock (it ends in its one host read);
  (b) the per-image path: nms.detections_per_image, metrics.match_detections per image, numpy ap_per_class over the
      concatenated rows, timed on the host clock ending in a device synchronise.

The detections are synthetic: per image 1-8 targets, several detections around each and 4000 background boxes, through
nms.detect_postprocess_classes (not timed).  Both paths are checked to give the same statistics before anything is
reported.  The card's name, power limit and SM clock are read in the same run.

    python tools/eval_times.py OUT_DIR [--reps 3]

Writes OUT_DIR/eval_times.json.  Needs a GPU."""
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

IMAGES, BATCH, SIZE, CONF, NMS, CAP, BACKGROUND = 444, 16, 512, 0.001, 0.5, 20000, 4000


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        name, pl, mx, sm = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit_w": float(pl), "sm_max_mhz": float(mx), "sm_mhz": float(sm)}
    except Exception as e:  # noqa: BLE001 -- report, do not fail the measurement
        return {"error": repr(e)[:200]}


def make_batches():
    import torch
    import helpers
    from rotate_yolov3_b200.nms import detect_postprocess_classes
    g = torch.Generator().manual_seed(0)
    batches = []
    for b0 in range(0, IMAGES, BATCH):
        bsz = min(BATCH, IMAGES - b0)
        ios, tg = [], []
        for b in range(bsz):
            nt = int(torch.randint(1, 9, (1,), generator=g))
            t = helpers.gen_boxes(nt, 10 * b0 + b, 400.0)
            t[:, :2] += 56.0
            near = t.repeat(6, 1)
            near[:, :2] += 0.1 * near[:, 2:4].max(1, keepdim=True).values * (torch.rand(len(near), 2, generator=g) - 0.5)
            near[:, 4] += 0.2 * (torch.rand(len(near), generator=g) - 0.5)
            boxes = torch.cat([near, helpers.gen_boxes(BACKGROUND, 7919 + b0 + b, float(SIZE))])
            io = torch.zeros(len(boxes), 7)
            io[:, :5] = boxes
            io[:, 5] = 0.002 + 0.99 * torch.rand(len(boxes), generator=g)
            io[:, 6] = 0.6 + 0.4 * torch.rand(len(boxes), generator=g)
            ios.append(io)
            tg.append(torch.cat([torch.full((nt, 1), float(b)), torch.zeros(nt, 1), t[:, 0:1] / SIZE, t[:, 1:2] / SIZE,
                                 t[:, 2:3] / SIZE, t[:, 3:4] / SIZE, t[:, 4:5]], 1))
        p = max(len(x) for x in ios)
        io = torch.stack([torch.cat([x, torch.zeros(p - len(x), 7)]) for x in ios]).cuda()
        batches.append((detect_postprocess_classes(io, CONF, NMS, CAP), torch.cat(tg).cuda(), (SIZE, SIZE)))
    torch.cuda.synchronize()
    return batches


def device_pass(batches):
    import torch
    from rotate_yolov3_b200.metrics import Evaluator
    ev = Evaluator(1, 0.5)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for res, targets, hw in batches:
        ev.add(res, targets, hw)
    e1.record()
    e1.synchronize()
    t0 = time.perf_counter()
    out = ev.compute()
    t1 = time.perf_counter()
    return out, e0.elapsed_time(e1) / len(batches), (t1 - t0) * 1e3


def per_image_pass(batches):
    import torch
    from ap_numpy import ap_per_class
    from rotate_yolov3_b200.metrics import match_detections
    from rotate_yolov3_b200.nms import detections_per_image
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    stats, seen = [], 0
    for res, targets, (height, width) in batches:
        for si, pred in enumerate(detections_per_image(res)):
            labels = targets[targets[:, 0] == si, 1:]
            tcls = labels[:, 0].tolist()
            seen += 1
            if pred is None:
                if tcls:
                    stats.append(([], np.zeros(0, np.float32), np.zeros(0, np.float32), tcls))
                continue
            correct = [0] * len(pred)
            if tcls:
                tbox = labels[:, 1:6].clone()
                tbox[:, [0, 2]] *= width
                tbox[:, [1, 3]] *= height
                correct = match_detections(pred, tbox, labels[:, 0])
            stats.append((correct, pred[:, 5].cpu().numpy(), pred[:, 7].cpu().numpy(), tcls))
    stats = [np.concatenate(x, 0) for x in zip(*stats)]
    p, r, ap, f1, ap_class = ap_per_class(*stats)
    nt = np.bincount(stats[3].astype(np.int64), minlength=1)
    torch.cuda.synchronize()
    return (p, r, ap, f1, ap_class, nt, seen), (time.perf_counter() - t0) * 1e3, len(stats[0])


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("out_dir")
    ap_.add_argument("--reps", type=int, default=3)
    args = ap_.parse_args()
    import torch
    batches = make_batches()
    device_pass(batches)                                  # warm-up: module loads, allocator, sort plans
    per_image_pass(batches)
    dev_runs, host_runs = [], []
    for _ in range(args.reps):
        got, add_ms, compute_ms = device_pass(batches)
        want, loop_ms, rows = per_image_pass(batches)
        dev_runs.append((add_ms, compute_ms))
        host_runs.append(loop_ms)
    p, r, ap, f1, cls, nt, seen = got
    wp, wr, wap, wf1, wcls, wnt, wseen = want
    assert np.array_equal(cls, wcls) and np.array_equal(nt, wnt) and seen == wseen
    assert np.array_equal(p, wp) and np.array_equal(r, wr) and np.array_equal(f1, wf1)
    assert np.all(np.abs(ap - wap) <= 1e-12 * np.abs(wap))
    add_ms = float(np.median([d[0] for d in dev_runs]))
    compute_ms = float(np.median([d[1] for d in dev_runs]))
    loop_ms = float(np.median(host_runs))
    result = {
        "gpu": gpu_info(), "torch": torch.__version__, "images": IMAGES, "batch": BATCH, "size": SIZE, "cap": CAP,
        "conf_thres": CONF, "rows": int(rows), "targets": int(nt.sum()), "ap": float(ap[0]),
        "evaluator_add_ms_per_batch": add_ms, "evaluator_compute_ms": compute_ms,
        "evaluator_pass_ms": add_ms * len(batches) + compute_ms, "per_image_pass_ms": loop_ms,
        "runs": {"device": dev_runs, "per_image": host_runs},
    }
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "eval_times.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
