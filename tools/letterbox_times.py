"""What letterboxing costs on the device, and what it saves detect.py.  All in one process, with the card's name and power
limit read in the same run:

* kernel time of ryolo_letterbox from CUDA events over CUDA-graph replays of 20 launches (no host overhead), at batch 1
  and 32, for 1024x768 and 1920x1080 sources to 608^2 and the 2x integer case 1216x912;
* achieved GB/s from the bytes the algorithm needs (uint8 source read + output write), against 3.35 TB/s (H100 SXM
  data sheet) and against a device-to-device copy moving the same number of bytes in the same process;
* detect.py's per-image loop at batch 1 (yolov3, 608, CUDA-graph forward, detect_postprocess_classes, the kept counts
  read back), alternating two paths image by image:
    host   cv2 letterbox + normalisation on the CPU (the reference's), fp32 upload, forward, postprocess;
    device pinned uint8 upload + letterbox on the device, forward, postprocess;
  and the host letterbox alone, with the CPU model and cv2's thread count.

    python tools/letterbox_times.py OUT_DIR [--images 40]

Writes OUT_DIR/letterbox_times.json.  Needs a GPU."""
import argparse
import json
import os
import platform
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCES = {"1024x768": (768, 1024), "1920x1080": (1080, 1920), "1216x912_2x": (912, 1216)}
HBM_TBS = 3.35


def cpu_name():
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                return line.split(":", 1)[1].strip()
    except OSError:
        pass
    return platform.processor() or "unknown (%s)" % platform.machine()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--images", type=int, default=40)
    a = ap.parse_args()
    sys.path[:0] = [REPO, os.path.join(REPO, "tests"), os.path.join(REPO, "tools")]
    import numpy as np
    import torch
    import helpers
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs, preprocess
    from rotate_yolov3_b200.nms import detect_postprocess_classes
    from se_step_times import gpu_info
    os.makedirs(a.out, exist_ok=True)
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_info(), "cpu": cpu_name(), "cpu_count": os.cpu_count(), "kernel": [], "detect_loop": {}}

    def graph_ms(fn, launches=20, reps=50):
        """device time per call of fn from CUDA events around replays of a graph of `launches` calls"""
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
    for name, (h, w) in SOURCES.items():
        for batch in (1, 32):
            imgs = [torch.from_numpy(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).to(dev) for _ in range(batch)]
            out = torch.empty((batch, 3, 608, 608), dtype=torch.float32, device=dev)
            ms = graph_ms(lambda: pkg.letterbox(imgs, 608, out=out))
            nbytes = batch * (h * w * 3 + 3 * 608 * 608 * 4)
            half = torch.empty(nbytes // 2, dtype=torch.uint8, device=dev)
            dst = torch.empty_like(half)
            copy_ms = graph_ms(lambda: dst.copy_(half))        # reads and writes nbytes / 2 each: nbytes moved
            kind = preprocess.resample_tables((h, w), preprocess.geometry((h, w), 608)[0])[0]
            row = {"source": name, "batch": batch, "kind": kind, "kernel_ms": ms, "bytes": nbytes, "gbs": nbytes / ms / 1e6, "copy_ms": copy_ms,
                   "copy_gbs": nbytes / copy_ms / 1e6}
            row["of_hbm"] = row["gbs"] / (HBM_TBS * 1e3)
            row["of_copy"] = row["gbs"] / row["copy_gbs"]
            res["kernel"].append(row)
            print(json.dumps(row), flush=True)
            del imgs, out, half, dst

    # detect.py per-image loop at batch 1
    try:
        import cv2
        res["cv2"] = {"version": cv2.__version__, "threads": cv2.getNumThreads()}
    except ImportError:
        cv2 = None
        res["cv2"] = "unavailable"
    model = pkg.Darknet(cfgs.yolov3_cfg(), {"context_factor": 1.0}, arc="default")
    helpers.init_darknet_weights(model, seed=1)
    model = model.to(dev).eval()
    model.use_cuda_graph = True

    def host_letterbox(img0):
        (nh, nw), (top, bottom, left, right), _ = preprocess.geometry(img0.shape[:2], 608)
        img = cv2.resize(img0, (nw, nh), interpolation=cv2.INTER_AREA) if (nh, nw) != img0.shape[:2] else img0
        img = cv2.copyMakeBorder(img, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(128, 128, 128))
        img = np.ascontiguousarray(img[:, :, ::-1].transpose(2, 0, 1), dtype=np.float32)
        img /= 255.0
        return img

    def post(io):
        return detect_postprocess_classes(io, 0.5, 0.5, 20000)["num_keep"].tolist()

    def host_path(img0):
        x = torch.from_numpy(host_letterbox(img0)).to(dev).unsqueeze(0)
        with torch.no_grad():
            return post(model(x)[0])

    pinned = {}

    def device_path(img0):
        buf = pinned.get(img0.shape)
        if buf is None:
            buf = pinned[img0.shape] = torch.empty(img0.shape, dtype=torch.uint8, pin_memory=True)
        buf.numpy()[...] = img0
        x, _ = pkg.letterbox([buf.to(dev, non_blocking=True)], 608)
        with torch.no_grad():
            return post(model(x)[0])

    for name, (h, w) in SOURCES.items():
        if name.endswith("_2x"):
            continue
        imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(4)]
        loop = {}
        if cv2 is not None:
            assert np.array_equal(host_letterbox(imgs[0]), pkg.letterbox([imgs[0]], 608)[0][0].cpu().numpy())
            paths = (("host", host_path), ("device", device_path))
            for _, fn in paths:                       # warm-up: plan build, graph capture, pinned buffers
                fn(imgs[0])
                fn(imgs[1])
            times = {k: [] for k, _ in paths}
            for i in range(a.images):
                for k, fn in (paths if i % 2 == 0 else paths[::-1]):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn(imgs[i % len(imgs)])
                    torch.cuda.synchronize()
                    times[k].append((time.perf_counter() - t0) * 1e3)
            lb = []
            for i in range(a.images):
                t0 = time.perf_counter()
                host_letterbox(imgs[i % len(imgs)])
                lb.append((time.perf_counter() - t0) * 1e3)
            for k, v in times.items():
                loop[k + "_ms_median"] = float(np.median(v))
                loop[k + "_ms_min"] = float(np.min(v))
            loop["host_letterbox_ms_median"] = float(np.median(lb))
        res["detect_loop"][name] = loop
        print(name, json.dumps(loop), flush=True)
    with open(os.path.join(a.out, "letterbox_times.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"gpu": res["gpu"], "cpu": res["cpu"], "cv2": res["cv2"]}))


if __name__ == "__main__":
    main()
