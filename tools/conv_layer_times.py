"""Where the bf16 training step's time goes: per conv shape, the forward (conv_igemm_kernel), weight-gradient
(conv_wgrad_kernel) and data-gradient (conv_igemm_kernel with the dgrad descriptor) launches of the batch-64 608x608
Darknet-53 step, each timed with CUDA events and set next to a torch.matmul bf16 GEMM of the same M x N x K on the same
card; then a torch.profiler breakdown of one eager step by kernel family and by kernel name.

    python tools/conv_layer_times.py OUT_DIR [--batch 64] [--iters 20]

Writes OUT_DIR/conv_layer_times.json and OUT_DIR/conv_layer_times.txt.  Needs a GPU; the plan is built the way
bench.py builds its default training step (same model, weights, images and targets)."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
from collections import OrderedDict

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))

MATMUL_BYTES = 1 << 30   # largest operand of the comparison GEMM; a longer M or K is shortened (the rate has saturated)


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        name, pl, mx, sm = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit_w": float(pl), "sm_max_mhz": float(mx), "sm_mhz": float(sm)}
    except Exception as e:  # noqa: BLE001 -- report, do not fail the measurement
        return {"error": repr(e)[:200]}


def round_up(x, m):
    return (x + m - 1) // m * m


def conv_bn(cout):
    return 256 if cout > 128 else (128 if cout > 64 else 64)


def event_time_us(fn, iters, warmup=3):
    import torch
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def matmul_rate(m, n, k, iters):
    """TFLOP/s of a bf16 torch.matmul [m, k] x [k, n]; the longest of m, k is shortened to keep operands <= 1 GB"""
    import torch
    big = max(m * k, k * n, m * n) * 2
    if big > MATMUL_BYTES:
        f = MATMUL_BYTES / big
        if m >= k:
            m = max(256, int(m * f) // 256 * 256)
        else:
            k = max(256, int(k * f) // 256 * 256)
    a = torch.randn(m, k, dtype=torch.bfloat16, device="cuda")
    b = torch.randn(k, n, dtype=torch.bfloat16, device="cuda")
    us = event_time_us(lambda: torch.matmul(a, b), iters)
    del a, b
    return 2.0 * m * n * k / (us * 1e-6) / 1e12, [m, n, k]


def family(name):
    if "conv_igemm" in name:
        return "conv_igemm"
    if "conv_wgrad" in name:
        return "conv_wgrad"
    if "bn_" in name:
        return "bn_*"
    if any(s in name for s in ("bce", "loss", "rows_", "obj_")):
        return "loss"
    if "ryolo" in name:
        return "other ryolo"
    return "framework"


def kernel_name(name):
    """the kernel's qualified name without the return type and the parameter list, at most 70 characters"""
    if name.startswith("void "):
        name = name[5:]
    depth = 0
    for i, ch in enumerate(name):         # cut at the parameter list, not at a '(' inside template arguments
        depth += ch == "<"
        depth -= ch == ">"
        if ch == "(" and depth == 0 and i > 0:
            name = name[:i]
            break
    return name if len(name) <= 70 else name[:67] + "..."


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)

    import torch
    import bench
    import helpers
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import _lib, cfgs
    from rotate_yolov3_b200.loss import compute_loss
    if not torch.cuda.is_available():
        raise SystemExit("conv_layer_times.py needs a GPU")
    dev = torch.device("cuda", 0)
    lib = _lib.lib
    B = args.batch

    net = pkg.Darknet(cfgs.yolov3_cfg(), dict(bench.TRAIN_HYP), arc="default")
    helpers.init_darknet_weights(net, seed=1)
    net.nc, net.hyp = 1, dict(bench.TRAIN_HYP)
    net = net.to(dev).train()
    net.use_cuda_graph = False
    x = torch.rand(B, 3, 608, 608, generator=torch.Generator().manual_seed(0)).to(dev)
    tg = bench.make_targets(B, 100).to(dev)

    def train_step():
        for p in net.parameters():
            p.grad = None
        ps = net(x)
        loss, _ = compute_loss(ps, tg.clone(), net, net.hyp)
        loss.backward()

    train_step()          # every plan buffer populated
    torch.cuda.synchronize()
    plan = net._tplan
    st = _lib.stream_ptr(dev)

    # ---- one row per distinct conv shape
    rows = OrderedDict()
    for blk in plan.blocks:
        h, w = blk.src.h, blk.src.w
        key = (blk.cin, blk.cout, blk.k, blk.stride, h, w, blk.is_head, blk.gsrc_acc if blk.gsrc is not None else None)
        if key in rows:
            rows[key]["count"] += 1
            rows[key]["layers"].append(blk.i)
            continue
        algo = 2.0 * B * blk.oh * blk.ow * blk.cout * blk.cin * blk.k * blk.k
        # GEMM geometry as the kernels run it
        if blk.s2d:
            gh, gw, taps, cin_eff = h // 2, w // 2, 4, blk.cin_eff
        else:
            gh, gw, taps, cin_eff = h, w, blk.k_eff * blk.k_eff, blk.cin_eff
        np_ = B * (gh + 2) * (gw + 2)
        bn_f = conv_bn(blk.cout)
        mma_f = 2.0 * round_up(np_, 128) * round_up(blk.cout, bn_f) * taps * round_up(cin_eff, 64)
        r = {"layers": [blk.i], "count": 1, "cin": blk.cin, "cout": blk.cout, "k": blk.k, "stride": blk.stride,
             "in_hw": [h, w], "s2d": bool(blk.s2d), "head": bool(blk.is_head), "bn_fwd": bn_f,
             "algo_gflop": algo / 1e9}
        x_ptr = blk.xs.data_ptr() if blk.s2d else blk.src.ptr
        if blk.is_head:
            fwd = (blk.fdesc, x_ptr, blk.pw, blk.bias_pad, blk.out)
        else:
            fwd = (blk.fdesc, x_ptr, blk.pw, plan.zero_bias, blk.z)

        def run_fwd(a=fwd):
            _lib.check(lib.ryolo_conv_bn_act_fwd(ctypes.byref(a[0]), ctypes.c_void_p(a[1]), _lib.ptr(a[2]), _lib.ptr(a[3]),
                                                 None, _lib.ptr(a[4]), st), "conv")
        r["fwd_us"] = event_time_us(run_fwd, args.iters)
        r["fwd_mma_gflop"] = mma_f / 1e9
        r["fwd_matmul_tflops"], r["fwd_matmul_mnk"] = matmul_rate(B * blk.oh * blk.ow, blk.cout,
                                                                  blk.cin * blk.k * blk.k, args.iters)

        dz = blk.dz if blk.is_head else blk.z
        if blk.s2d:
            wg = (dz, blk.zcs, blk.cout_pad, blk.xs.data_ptr(), blk.xs_cs, blk.cin_pad, gh, gw, 2)
        else:
            if blk.stride == 2:
                dz = blk.dz_up
            wg = (dz, blk.zcs, blk.cout_pad, blk.src.ptr, blk.src.cs, blk.cin_pad, gh, gw, blk.k_eff)

        def run_wgrad(a=wg, dw=blk.dw):
            _lib.check(lib.ryolo_conv_wgrad(_lib.ptr(a[0]), a[1], a[2], ctypes.c_void_p(a[3]), a[4], a[5], B, a[6], a[7],
                                            a[8], _lib.ptr(dw), st), "wgrad")
        r["wgrad_us"] = event_time_us(run_wgrad, args.iters)
        r["wgrad_mma_gflop"] = 2.0 * round_up(blk.cout_pad, 128) * blk.cin_pad * taps * round_up(np_, 64) / 1e9
        r["wgrad_matmul_tflops"], r["wgrad_matmul_mnk"] = matmul_rate(blk.cout, blk.cin * blk.k * blk.k,
                                                                      B * blk.oh * blk.ow, args.iters)

        if blk.i > 0:
            bn_d = conv_bn(cin_eff)
            r["dgrad_mma_gflop"] = 2.0 * round_up(np_, 128) * round_up(cin_eff, bn_d) * taps * round_up(blk.cout, 64) / 1e9
            r["bn_dgrad"] = bn_d
            if blk.s2d:
                def run_dgrad(blk=blk, dz=dz):
                    _lib.check(lib.ryolo_conv_bn_act_fwd(ctypes.byref(blk.ddesc), _lib.ptr(dz), _lib.ptr(blk.pwd),
                                                         _lib.ptr(plan.zero_bias), None, _lib.ptr(blk.dxs), st),
                               "dgrad s2d")
            else:
                def run_dgrad(blk=blk, dz=dz):
                    gp = blk.gsrc.ptr
                    blk.ddesc.has_residual = int(blk.gsrc_acc)
                    _lib.check(lib.ryolo_conv_bn_act_fwd(ctypes.byref(blk.ddesc), _lib.ptr(dz), _lib.ptr(blk.pwd),
                                                         _lib.ptr(plan.zero_bias),
                                                         ctypes.c_void_p(gp) if blk.gsrc_acc else None,
                                                         ctypes.c_void_p(gp), st), "dgrad")
            r["dgrad_us"] = event_time_us(run_dgrad, args.iters)
            r["dgrad_matmul_tflops"], r["dgrad_matmul_mnk"] = matmul_rate(B * h * w, blk.cin, blk.cout * blk.k * blk.k,
                                                                          args.iters)
        rows[key] = r
    torch.cuda.synchronize()
    for r in rows.values():
        for kind in ("fwd", "wgrad", "dgrad"):
            if kind + "_us" in r:
                s = r[kind + "_us"] * 1e-6
                r[kind + "_algo_tflops"] = r["algo_gflop"] * 1e-3 / s
                r[kind + "_mma_tflops"] = r[kind + "_mma_gflop"] * 1e-3 / s
                r[kind + "_of_matmul"] = r[kind + "_algo_tflops"] / r[kind + "_matmul_tflops"]
    clocks = gpu_info()     # read while the card is warm from the launches above

    # ---- one eager step under torch.profiler, device time by kernel family
    from torch.profiler import ProfilerActivity, profile
    train_step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        train_step()
        torch.cuda.synchronize()
    fam, kern = {}, {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0.0)
        if t <= 0:
            continue
        f = family(ev.key)
        fam[f] = fam.get(f, 0.0) + t / 1e3
        name = kernel_name(ev.key)
        k = kern.setdefault(name, {"family": f, "calls": 0, "ms": 0.0})
        k["calls"] += ev.count
        k["ms"] += t / 1e3
    kernel_ms = sum(fam.values())
    # per kernel name: every kernel of the loss family and every ryolo kernel, plus the largest framework ones
    shown = [(n, k) for n, k in sorted(kern.items(), key=lambda kv: -kv[1]["ms"])
             if k["family"] != "framework" or k["ms"] >= 0.01 * kernel_ms]

    totals = {k: sum(r.get(k + "_us", 0.0) * r["count"] for r in rows.values()) / 1e3 for k in ("fwd", "wgrad", "dgrad")}
    res = {"gpu": clocks, "batch": B, "iters": args.iters, "rows": list(rows.values()),
           "gemm_ms_from_rows": totals, "profile_ms_by_family": fam, "profile_ms_by_kernel": kern,
           "profile_kernel_ms": kernel_ms}
    with open(os.path.join(args.out_dir, "conv_layer_times.json"), "w") as f:
        json.dump(res, f, indent=1)

    lines = ["%s, power limit %s W, SM clock %s MHz (max %s) -- batch %d, %d launches per timing" %
             (clocks.get("name"), clocks.get("power_limit_w"), clocks.get("sm_mhz"), clocks.get("sm_max_mhz"), B,
              args.iters)]
    hdr = "%-22s %3s | %-28s | %-28s | %-28s" % ("layer shape", "n", "fwd us  TF/s alg mma  %mm", "wgrad us TF/s alg mma %mm",
                                                 "dgrad us TF/s alg mma %mm")
    lines += [hdr, "-" * len(hdr)]
    for r in rows.values():
        shape = "%dx%d k%d%s %d->%d" % (r["in_hw"][0], r["in_hw"][1], r["k"], "s2" if r["stride"] == 2 else "",
                                        r["cin"], r["cout"])
        cells = []
        for kind in ("fwd", "wgrad", "dgrad"):
            if kind + "_us" in r:
                cells.append("%8.1f %4.0f %4.0f %4.0f" % (r[kind + "_us"], r[kind + "_algo_tflops"], r[kind + "_mma_tflops"],
                                                        100 * r[kind + "_of_matmul"]))
            else:
                cells.append("%-28s" % "")
        lines.append("%-22s %3d | %s | %s | %s" % (shape + (" head" if r["head"] else ""), r["count"], *cells))
    lines.append("")
    lines.append("sum over the step (us x count): fwd %.1f ms, wgrad %.1f ms, dgrad %.1f ms" %
                 (totals["fwd"], totals["wgrad"], totals["dgrad"]))
    lines.append("one eager step under torch.profiler, device time %.1f ms:" % kernel_ms)
    for k, v in sorted(fam.items(), key=lambda kv: -kv[1]):
        lines.append("  %-12s %8.1f ms  %5.1f %%" % (k, v, 100 * v / kernel_ms))
    lines.append("by kernel (every ryolo kernel; framework kernels from 1 %% of the step):")
    lines.append("  %-70s %-12s %6s %9s %9s" % ("kernel", "family", "calls", "ms", "us/call"))
    for n, k in shown:
        lines.append("  %-70s %-12s %6d %9.3f %9.1f" % (n, k["family"], k["calls"], k["ms"], 1e3 * k["ms"] / max(k["calls"], 1)))
    txt = "\n".join(lines)
    with open(os.path.join(args.out_dir, "conv_layer_times.txt"), "w") as f:
        f.write(txt + "\n")
    print(txt)


if __name__ == "__main__":
    main()
