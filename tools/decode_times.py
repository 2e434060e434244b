"""What decoding JPEG on the device costs, and what it saves the training input path.  All in one process, with the
card's name, power limit and clock read in the same run.  Per batch of 64 images, for the reference's HRSC sample
(1167 x 821; the file itself for 4:2:0 without restarts, cv2 re-encodes of its pixels at q90 otherwise) and a
1920 x 1080 q95 frame, 4:2:0 and 4:4:4, without restart markers and with one per MCU row:

* device time of ryolo_jpeg_decode from CUDA events over CUDA-graph replays, split into the entropy stage and the
  IDCT / upsampling / colour stage, and the whole call;
* the host time of cv2.imread on the same files (from a temporary directory), with 1 and 8 threads;
* bytes staged (job and code tables plus compressed bytes) against the decoded pixels the raw-pixel path uploads;
* decode_images -> train_batch against cv2.imread -> train_batch, end to end per batch (host clock, synchronised),
  alternating the two.

    python tools/decode_times.py OUT_DIR [--batch 64] [--reps 5]

Writes OUT_DIR/decode_times.json.  Needs a GPU."""
import argparse
import json
import os
import random
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HYP = {"degrees": 5.0, "translate": 0.1, "scale": 0.2, "shear": 0.0, "noise": 0.0, "gamma": 0.2, "blur": 0.0,
       "hsv_s": 0.5, "hsv_v": 0.3, "grayscale": 0.0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    sys.path[:0] = [REPO, os.path.join(REPO, "tests"), os.path.join(REPO, "tools")]
    import cv2
    import numpy as np
    import torch
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200.decode import Batch
    from jpeg_cases import encode, hrsc, picture
    from se_step_times import gpu_info
    if not torch.cuda.is_available():
        raise SystemExit("decode_times needs a GPU")
    os.makedirs(a.out, exist_ok=True)
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_info(), "cpu_count": os.cpu_count(), "cv2": cv2.__version__, "batch": a.batch, "cases": []}

    def graph_ms(fn, launches=5, reps=10):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            fn()
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(launches):
                fn()
        g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / (launches * reps)

    hr = hrsc()
    hr_pixels = cv2.imdecode(np.frombuffer(hr, np.uint8), cv2.IMREAD_COLOR)
    hd_pixels = picture(11, 1080, 1920)
    cases = []
    for size, px in (("hrsc_1167x821", hr_pixels), ("1920x1080", hd_pixels)):
        for s in ("420", "444"):
            row = -(-px.shape[1] // (16 if s == "420" else 8))
            for rst in (0, row):
                if size.startswith("hrsc") and s == "420" and rst == 0:
                    blob = hr
                else:
                    blob = encode(px, 90 if size.startswith("hrsc") else 95, s, restart=rst)
                cases.append(("%s_%s_rst%d" % (size, s, rst), blob))
    labs = [np.array([[0, 0.5, 0.5, 0.2, 0.1, 0.3]], np.float32)] * a.batch
    with tempfile.TemporaryDirectory() as tmp:
        for name, blob in cases:
            paths = []
            for i in range(a.batch):
                p = os.path.join(tmp, "%s_%d.jpg" % (name, i))
                with open(p, "wb") as f:
                    f.write(blob)
                paths.append(p)
            blobs = [np.fromfile(p, np.uint8) for p in paths]
            batch = Batch(blobs, dev)
            batch.decode()
            imgs, routes = batch.finish()
            assert all(r == "device" for r in routes), routes[:2]
            want = cv2.imread(paths[0])
            assert np.array_equal(imgs[0].cpu().numpy(), want) and np.array_equal(imgs[-1].cpu().numpy(), want), name
            row = {"case": name, "bytes_per_file": len(blob), "hw": list(want.shape[:2]),
                   "nchunks": batch.lay.nchunks, "nsegs": batch.lay.nsegs}
            row["entropy_ms"] = graph_ms(lambda: batch.decode(1))
            row["pixels_ms"] = graph_ms(lambda: batch.decode(2))
            row["decode_ms"] = graph_ms(lambda: batch.decode(3))
            row["staged_bytes"] = batch.staged_bytes
            row["raw_pixel_bytes"] = int(sum(im.numel() for im in imgs))
            for threads in (1, 8):
                cv2.imread(paths[0])
                ts = []
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    if threads == 1:
                        for p in paths:
                            cv2.imread(p)
                    else:
                        with ThreadPoolExecutor(threads) as ex:
                            list(ex.map(cv2.imread, paths))
                    ts.append(time.perf_counter() - t0)
                row["imread_ms_%dthreads" % threads] = 1e3 * min(ts)
            ends = {"device": [], "host": []}
            for rep in range(a.reps + 1):
                for path in ("device", "host"):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if path == "device":
                        src, _ = pkg.decode_images([np.fromfile(p, np.uint8) for p in paths], device=dev)
                    else:
                        src = [cv2.imread(p) for p in paths]
                    x, _, _ = pkg.train_batch(src, labs, HYP, new_shape=608, rng=random.Random(rep))
                    torch.cuda.synchronize()
                    if rep:
                        ends[path].append(1e3 * (time.perf_counter() - t0))
            row["train_batch_from_decode_images_ms"] = min(ends["device"])
            row["train_batch_from_imread_ms"] = min(ends["host"])
            res["cases"].append(row)
            print(json.dumps(row), flush=True)
            del batch, imgs
    with open(os.path.join(a.out, "decode_times.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"gpu": res["gpu"], "cpu_count": res["cpu_count"]}))


if __name__ == "__main__":
    main()
