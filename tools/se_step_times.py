"""What the squeeze-excitation blocks cost: each SE kernel at the batch-64 608 x 608 shapes (76^2 x 256, 38^2 x 512,
19^2 x 1024), timed with CUDA events over 50 launches and set next to a device-to-device copy measured in the same process;
then the network forward + backward of cfg/ICDAR/yolov3_608_se.cfg against cfg/ICDAR/yolov3_608.cfg (same anchor file,
same batch, CUDA graphs on, a fixed head cotangent in place of the loss) alternated three times, and the eval forward of
both graphs at batch 32.  The card's name, power limit and SM clock are read in the same run.

    python tools/se_step_times.py OUT_DIR [--batch 64] [--iters 50] [--train-batch 32]

Writes OUT_DIR/se_step_times.json.  Needs a GPU.  The training steps run at --train-batch (32): both graphs stay
resident so that their steps alternate, and at batch 64 the two plans together do not fit in 80 GB."""
import argparse
import gc
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
REF_CFG = os.path.join(REPO, "tests", "golden", "reference_cfg")


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


def kernel_times(batch, iters):
    import torch
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import layout as L
    lib, dev = pkg._lib.lib, torch.device("cuda")
    P, st = pkg._lib.ptr, pkg._lib.stream_ptr(dev)
    rows = []
    for hw, c in ((76, 256), (38, 512), (19, 1024)):
        cr = c // 16
        x = L.alloc_padded(batch, hw, hw, c, dev)
        x[:, 1:-1, 1:-1].normal_()
        u, gu, gx = torch.zeros_like(x), torch.randn_like(x), torch.randn_like(x)
        gu[:, 0] = gu[:, -1] = gu[:, :, 0] = gu[:, :, -1] = 0
        w1, w2 = torch.randn(cr, c, device=dev) * 0.05, torch.randn(c, cr, device=dev) * 0.05
        f = lambda n: torch.zeros(n, dtype=torch.float32, device=dev)     # noqa: E731
        m, p, s, ds, dm, gw1, gw2 = f(batch * c), f(batch * cr), f(batch * c), f(batch * c), f(batch * c), f(c * cr), f(c * cr)
        ws = torch.empty(lib.ryolo_se_workspace_bytes(batch, hw, hw, c, cr), dtype=torch.uint8, device=dev)

        def fwd():
            pkg._lib.check(lib.ryolo_se_fwd(P(x), c, P(u), c, batch, hw, hw, c, P(w1), P(w2), cr, P(m), P(p), P(s), P(ws),
                                            ws.numel(), st), "se_fwd")

        def bwd():
            pkg._lib.check(lib.ryolo_se_bwd(P(gu), c, P(x), c, P(gx), c, 1, batch, hw, hw, c, P(w1), P(w2), cr, P(m), P(p),
                                            P(s), P(ds), P(dm), P(gw1), P(gw2), P(ws), ws.numel(), st), "se_bwd")
        act = x.numel() * 2                          # bytes of one padded activation
        dst = torch.empty_like(x)
        t_copy = event_ms(lambda: dst.copy_(x), iters)
        t_f, t_b = event_ms(fwd, iters), event_ms(bwd, iters)
        # bytes the algorithm moves: forward reads x twice (pool, scale) and writes u; backward reads gu and x (reduce),
        # gu again and gx, and writes gx
        rows.append({"shape": "%d^2 x %d" % (hw, c), "batch": batch, "activation_mb": act / 1e6,
                     "copy_ms": t_copy, "copy_gbps": 2 * act / t_copy / 1e6,
                     "fwd_ms": t_f, "fwd_gbps": 3 * act / t_f / 1e6, "bwd_ms": t_b, "bwd_gbps": 5 * act / t_b / 1e6})
        print(json.dumps(rows[-1]), flush=True)
        del x, u, gu, gx, dst, ws
        torch.cuda.empty_cache()
    return rows


def build(cfg, seed):
    import rotate_yolov3_b200 as pkg
    from helpers import init_darknet_weights
    cwd = os.getcwd()
    os.chdir(REF_CFG)
    try:
        m = pkg.Darknet(cfg, {"context_factor": 1.0}, arc="default")
    finally:
        os.chdir(cwd)
    init_darknet_weights(m, seed=seed)
    return m.cuda()


def step_fn(m, x):
    import torch
    m.train()
    m.use_cuda_graph = True
    gs = None

    def run():
        nonlocal gs
        ps = m(x)
        if gs is None:
            gs = [torch.randn(p.shape, device=x.device) for p in ps]
        sum((p * g).sum() for p, g in zip(ps, gs)).backward()
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--train-batch", type=int, default=32)
    a = ap.parse_args()
    import torch
    os.makedirs(a.out, exist_ok=True)
    res = {"gpu": gpu_info()}
    print(json.dumps(res["gpu"]), flush=True)
    res["kernels"] = kernel_times(a.batch, a.iters)
    # training step: SE graph vs plain graph
    # both graphs stay resident so that their steps can alternate: at batch 64 the two plans together exceed 80 GB
    batch = a.train_batch
    se, plain = build("cfg/ICDAR/yolov3_608_se.cfg", 1), build("cfg/ICDAR/yolov3_608.cfg", 1)
    x = torch.rand(batch, 3, 608, 608, device="cuda")
    f_se, f_plain = step_fn(se, x), step_fn(plain, x)
    res["train_batch"] = batch
    pairs = []
    for _ in range(3):
        pairs.append({"se_ms": event_ms(f_se, 10), "plain_ms": event_ms(f_plain, 10)})
        print(json.dumps(pairs[-1]), flush=True)
    res["train_step"] = pairs
    res["train_peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
    del se, plain, x, f_se, f_plain
    gc.collect()
    torch.cuda.empty_cache()
    # eval forward at batch 32
    ev = []
    se, plain = build("cfg/ICDAR/yolov3_608_se.cfg", 2).eval(), build("cfg/ICDAR/yolov3_608.cfg", 2).eval()
    se.use_cuda_graph = plain.use_cuda_graph = True
    x = torch.rand(32, 3, 608, 608, device="cuda")
    with torch.no_grad():
        for _ in range(3):
            ev.append({"se_ms": event_ms(lambda: se(x), 20), "plain_ms": event_ms(lambda: plain(x), 20)})
            print(json.dumps(ev[-1]), flush=True)
    res["eval_b32"] = ev
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "se_step_times.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k not in ("kernels",)}), flush=True)


if __name__ == "__main__":
    main()
