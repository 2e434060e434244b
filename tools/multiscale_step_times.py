"""What the reference's changing shapes cost: the multi-scale training loop of train.py:239-287 (an image size drawn every
10 batches; here the fixed sequence 768 -> 448 -> 608 -> 768 -> 512 for base size 608) at batch 64 on the yolov3 graph
with CUDA graphs on (as bench.py runs the step), and detect.py --multi-scale (two sizes alternating on every image,
detect.py:53-99) at batch 1.  Every step is timed on its own (host clock around work that ends in a device
synchronise), so the first step at a shape (plan build, weight packing, graph capture) and a revisit show separately;
peak max_memory_allocated is read after each step.  A CUDA out-of-memory error is recorded with the step it ended,
and ends that loop.  The card's name, power limit and SM clock are read in the same run.

    python tools/multiscale_step_times.py OUT_DIR [--tree DIR] [--batch 64] [--per-size 10] [--images 20]

--tree: the repository tree whose package is measured (default: this one; another checkout, built, to measure the
commit before it).  Writes OUT_DIR/multiscale_step_times_<label>.json.  Needs a GPU."""
import argparse
import gc
import json
import os
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TRAIN_SIZES = (768, 448, 608, 768, 512)
DETECT_SIZES = (512, 704)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--tree", default=REPO)
    ap.add_argument("--label", default="new")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--per-size", type=int, default=10)
    ap.add_argument("--images", type=int, default=20)
    a = ap.parse_args()
    sys.path[:0] = [os.path.abspath(a.tree), REPO, os.path.join(REPO, "tests"), os.path.join(REPO, "tools")]
    import torch
    import bench
    import helpers
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    from rotate_yolov3_b200.loss import compute_loss
    from se_step_times import gpu_info
    assert os.path.abspath(pkg.__file__).startswith(os.path.abspath(a.tree)), pkg.__file__
    os.makedirs(a.out, exist_ok=True)
    res = {"label": a.label, "gpu": gpu_info(), "batch": a.batch, "train_sizes": TRAIN_SIZES, "per_size": a.per_size}
    print(json.dumps(res), flush=True)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    net = pkg.Darknet(cfgs.yolov3_cfg(), dict(bench.TRAIN_HYP), arc="default")
    helpers.init_darknet_weights(net, seed=1)
    net.nc, net.hyp = 1, dict(bench.TRAIN_HYP)
    net = net.cuda().train()
    net.use_cuda_graph = True
    pg_w = [p for n, p in net.named_parameters() if "Conv2d.weight" in n]
    pg_o = [p for n, p in net.named_parameters() if "Conv2d.weight" not in n]
    opt = torch.optim.SGD([{"params": pg_o}, {"params": pg_w, "weight_decay": 4.569e-4}], lr=1e-4, momentum=0.97,
                          nesterov=True, fused=True)
    tg = bench.make_targets(a.batch, 100).cuda()
    torch.cuda.reset_peak_memory_stats()
    rows, seen = [], set()
    for si, s in enumerate(TRAIN_SIZES):
        x = torch.rand(a.batch, 3, s, s, generator=torch.Generator().manual_seed(si)).cuda()
        for k in range(a.per_size):
            def step():
                opt.zero_grad(set_to_none=True)
                loss, _ = compute_loss(net(x), tg.clone(), net, net.hyp)
                loss.backward()
                opt.step()
            row = {"size": s, "k": k, "first_visit": k == 0 and s not in seen}
            try:
                row["ms"] = timed(step)
            except torch.OutOfMemoryError as e:
                row["oom"] = str(e).splitlines()[0][:300]
                rows.append(row)
                print(json.dumps(row), flush=True)
                break
            row["peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
            # after a first visit, the growth of this beyond the pool is what the new plan holds for itself
            row["allocated_gb"] = torch.cuda.memory_allocated() / 1e9
            row["pool_gb"] = sum(p.nbytes for p in getattr(net, "_pools", {}).values()) / 1e9
            rows.append(row)
            print(json.dumps(row), flush=True)
        seen.add(s)
        if rows and "oom" in rows[-1]:
            break
    res["train"] = rows
    res["train_peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
    del net, opt, x
    gc.collect()              # a model and its plans reference each other
    torch.cuda.empty_cache()

    det = pkg.Darknet(cfgs.yolov3_cfg(), {"context_factor": 1.0}, arc="default")
    helpers.init_darknet_weights(det, seed=2)
    det = det.cuda().eval()
    det.use_cuda_graph = True
    torch.cuda.reset_peak_memory_stats()
    drows = []
    with torch.no_grad():
        for i in range(a.images):
            s = DETECT_SIZES[i % 2]
            x = torch.rand(1, 3, s, s, generator=torch.Generator().manual_seed(i)).cuda()
            drows.append({"image": i, "size": s, "ms": timed(lambda: det(x))})
            print(json.dumps(drows[-1]), flush=True)
    res["detect"] = drows
    res["detect_peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "multiscale_step_times_%s.json" % a.label), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
