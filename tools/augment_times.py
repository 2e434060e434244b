"""What the training augmentation costs on the device and on the host.  All in one process, with the card's name and
power limit read in the same run:

* device time per batch of ``train_batch``'s launches (pre-resize, letterbox, warp with the image maximum, finish)
  at 64 x (1024x768 -> 608^2) and 64 x (1920x1080 -> 608^2), every transform forced on (affine, gamma, HSV, both
  flips), CUDA sources, from CUDA events over CUDA-graph replays of 10 batches (no host overhead);
* the bytes the stages read and write, and a device-to-device copy of the same number of bytes in the same process;
* the reference's host chain per image for the same transforms (cv2 INTER_LINEAR pre-resize, letterbox, warpAffine,
  numpy gamma, cv2/numpy HSV, flips, BGR->RGB, /255) on this machine's CPU, one image at a time, with cv2's thread
  count;
* the whole ``train_batch`` call per image from host images and from CUDA images, and its host part split into the
  draws with the plan and label rows, the copy of the sources into pinned memory, and their upload.

    python tools/augment_times.py OUT_DIR [--images 16]

Writes OUT_DIR/augment_times.json.  Needs a GPU."""
import argparse
import json
import os
import random
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCES = {"1024x768": (768, 1024), "1920x1080": (1080, 1920)}
BATCH = 64
HBM_TBS = 3.35


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--images", type=int, default=16)
    a = ap.parse_args()
    sys.path[:0] = [REPO, os.path.join(REPO, "tools")]
    import cv2
    import numpy as np
    import torch
    import rotate_yolov3_b200 as pkg  # noqa: F401
    from rotate_yolov3_b200 import augment
    from letterbox_times import cpu_name
    from se_step_times import gpu_info
    os.makedirs(a.out, exist_ok=True)
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_info(), "cpu": cpu_name(), "cpu_count": os.cpu_count(),
           "cv2": {"version": cv2.__version__, "threads": cv2.getNumThreads()}, "device": [], "host": []}
    hyp = {"degrees": 5.0, "translate": 0.1, "scale": 0.1, "shear": 0.0, "noise": 0.01, "gamma": 0.2, "blur": 1.3,
           "hsv_s": 0.5, "hsv_v": 0.3, "grayscale": 0.3}
    rec = {"gray_alpha": 1.0, "affine": (3.7, 1.06, 0.04, -0.03), "noise": False, "gamma": 1.13, "blur": False,
           "hsv": (1.21, 0.86), "hflip": True, "vflip": True, "grayscale": False}

    def graph_free_ms(fn, reps=5):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    def graph_ms(fn, launches=10, reps=20):
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

    rng = np.random.default_rng(0)
    lab = np.array([[0, 0.5, 0.5, 0.2, 0.1, 0.3], [1, 0.3, 0.6, 0.1, 0.05, -0.7]], np.float32)
    for name, (h, w) in SOURCES.items():
        host = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(BATCH)]
        imgs = [torch.from_numpy(im).to(dev) for im in host]
        out = torch.empty((BATCH, 3, 608, 608), dtype=torch.float32, device=dev)
        plan, targets = augment.batch_plan([(h, w)] * BATCH, [lab] * BATCH, [rec] * BATCH, 608, "square")
        launch, _, keep = augment._stage(imgs, plan, targets, (608, 608), out, torch.float32, dev)
        ms = graph_ms(launch)
        hp, wp = plan[0][1]
        px = 608 * 608 * 3
        # source read, pre-resized image written and read, letterboxed image written, warp read and write, the row
        # maxima written and read (608 bytes each way), finish read and fp32 write
        nbytes = BATCH * (h * w * 3 + 2 * hp * wp * 3 + px + 2 * px + 2 * 608 + px + 4 * px)
        half = torch.empty(nbytes // 2, dtype=torch.uint8, device=dev)
        dst = torch.empty_like(half)
        copy_ms = graph_ms(lambda: dst.copy_(half))
        row = {"source": name, "batch": BATCH, "pre_resized": [hp, wp], "device_ms": ms, "bytes": nbytes,
               "gbs": nbytes / ms / 1e6, "copy_ms": copy_ms, "copy_gbs": nbytes / copy_ms / 1e6,
               "images_per_s": BATCH / ms * 1e3}
        row["of_hbm"] = row["gbs"] / (HBM_TBS * 1e3)
        row["of_copy"] = row["gbs"] / row["copy_gbs"]
        # the whole call, per image: from host images (pixels staged in pinned memory and uploaded) and from CUDA
        # images (job tables and targets only); and where the host part goes
        def wall_ms(srcs, reps=3):
            augment.train_batch(srcs, [lab] * BATCH, hyp, out=out)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(reps):
                augment.train_batch(srcs, [lab] * BATCH, hyp, out=out)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) / (reps * BATCH) * 1e3

        row["train_batch_wall_ms_per_image"] = wall_ms(host)
        row["train_batch_wall_ms_per_image_cuda_sources"] = wall_ms(imgs)
        t0 = time.perf_counter()
        for _ in range(3):
            r = random.Random(1)
            draws = [augment.draw(hyp, r) for _ in range(BATCH)]
            augment.batch_plan([(h, w)] * BATCH, [lab] * BATCH, draws, 608, "square")
        row["draws_plan_labels_ms_per_image"] = (time.perf_counter() - t0) / (3 * BATCH) * 1e3
        pinned = torch.empty(BATCH * h * w * 3, dtype=torch.uint8, pin_memory=True)
        stage = pinned.numpy()
        t0 = time.perf_counter()
        for _ in range(3):
            for k, im in enumerate(host):
                stage[k * h * w * 3:(k + 1) * h * w * 3] = im.reshape(-1)
        row["pinned_staging_ms_per_image"] = (time.perf_counter() - t0) / (3 * BATCH) * 1e3
        devbuf = torch.empty_like(pinned, device=dev)
        row["h2d_upload_ms_per_image"] = graph_free_ms(lambda: devbuf.copy_(pinned, non_blocking=True)) / BATCH
        row["h2d_gbs"] = pinned.numel() / (row["h2d_upload_ms_per_image"] * BATCH) / 1e6
        del pinned, stage, devbuf
        res["device"].append(row)
        print(json.dumps(row), flush=True)
        del imgs, out, half, dst, keep

        # the reference's host chain, one image at a time
        def host_chain(img):
            r = 608 / max(img.shape)
            if r < 1:
                img = cv2.resize(img, (int(img.shape[1] * r), int(img.shape[0] * r)), interpolation=cv2.INTER_LINEAR)
            (nh, nw), (top, bottom, left, right), _ = pkg.preprocess.geometry(img.shape[:2], 608)
            if (nh, nw) != img.shape[:2]:
                img = cv2.resize(img, (nw, nh), interpolation=cv2.INTER_AREA)
            img = cv2.copyMakeBorder(img, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(128, 128, 128))
            M = augment.affine_matrix(rec["affine"], img.shape[:2])
            img = cv2.warpAffine(img, M[:2], dsize=(608, 608), flags=cv2.INTER_AREA, borderValue=(128, 128, 128))
            img = np.uint8(np.power(img / float(np.max(img)), rec["gamma"]) * np.max(img))
            hsv = cv2.cvtColor(img, cv2.COLOR_BGR2HSV)
            S, V = hsv[:, :, 1].astype(np.float32), hsv[:, :, 2].astype(np.float32)
            S *= rec["hsv"][0]
            V *= rec["hsv"][1]
            hsv[:, :, 1] = S.clip(None, 255)
            hsv[:, :, 2] = V
            cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR, dst=img)
            img = np.flipud(np.fliplr(img))
            x = np.ascontiguousarray(img[:, :, ::-1].transpose(2, 0, 1), dtype=np.float32)
            x /= 255.0
            return x

        host_chain(host[0])
        t0 = time.perf_counter()
        for im in host[:a.images]:
            host_chain(im)
        ms_img = (time.perf_counter() - t0) / a.images * 1e3
        hrow = {"source": name, "host_chain_ms_per_image": ms_img, "images_per_s_one_thread": 1e3 / ms_img}
        res["host"].append(hrow)
        print(json.dumps(hrow), flush=True)
    with open(os.path.join(a.out, "augment_times.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"gpu": res["gpu"], "cpu": res["cpu"], "cpu_count": res["cpu_count"], "cv2": res["cv2"]}))


if __name__ == "__main__":
    main()
