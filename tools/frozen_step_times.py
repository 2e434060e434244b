"""What a training step costs when part of the network is frozen: the whole step (forward, compute_loss, backward and the
fused SGD step) of the yolov3 graph at batch 64 x 608 x 608, with every parameter trainable and under the three masks of
the reference's train.py: --transfer (the head convolutions, p.shape[0] == nf), --prebias (the head biases,
p.numel() == nf) and the frozen backbone (blocks >= 75 train).  CUDA graphs off and on.  The masks alternate in one
process, each round runs every mask in turn; a mask switch re-captures the graphs, so each mask's first two steps of a
round are not timed.  Also the bias-only head gradient kernel against the full head-gradient conversion at the three
head shapes.  The card's name, power limit and SM clock are read in the same run.

    python tools/frozen_step_times.py OUT_DIR [--batch 64] [--steps 10] [--rounds 3]

Writes OUT_DIR/frozen_step_times.json.  Needs a GPU."""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "tools"))

from se_step_times import event_ms, gpu_info  # noqa: E402


def masks(net):
    """requires_grad of every parameter, by the rules of reference train.py:120-135 and :215-220"""
    nf = int(net.module_defs[net.yolo_layers[0] - 1]["filters"])
    named = list(net.named_parameters())
    return {"full": [True] * len(named),
            "transfer": [p.shape[0] == nf for _, p in named],
            "prebias": [p.numel() == nf for _, p in named],
            "cutoff75": [int(n.split(".")[1]) >= 75 for n, _ in named]}


def head_kernels(batch, iters):
    """ryolo_head_bias_grad (reads the cotangent) against ryolo_head_grad_nchw_to_padded (reads it, writes bf16 dz)"""
    import torch
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import layout as L
    lib, dev = pkg._lib.lib, torch.device("cuda")
    P, st = pkg._lib.ptr, pkg._lib.stream_ptr(dev)
    c, rows = 504, []
    for n in (19, 38, 76):
        g = torch.randn(batch, c, n, n, device=dev)
        dst = L.alloc_padded(batch, n, n, 512, dev)
        bias = torch.zeros(c, device=dev)
        t_bias = event_ms(lambda: pkg._lib.check(lib.ryolo_head_bias_grad(P(g), batch, c, n, n, P(bias), st), "hb"), iters)
        t_full = event_ms(lambda: pkg._lib.check(lib.ryolo_head_grad_nchw_to_padded(P(g), batch, c, n, n, P(dst), 512,
                                                                                    P(bias), st), "hg"), iters)
        rd = g.numel() * 4
        rows.append({"shape": "%d x %d x %d^2" % (batch, c, n), "cotangent_mb": rd / 1e6,
                     "bias_only_ms": t_bias, "bias_only_gbps": rd / t_bias / 1e6,
                     "full_ms": t_full, "full_gbps": (rd + batch * n * n * c * 2) / t_full / 1e6})
        print(json.dumps(rows[-1]), flush=True)
        del g, dst
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    import bench
    import helpers
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    from rotate_yolov3_b200.loss import compute_loss
    os.makedirs(a.out, exist_ok=True)
    res = {"gpu": gpu_info(), "batch": a.batch}
    print(json.dumps(res["gpu"]), flush=True)
    res["head_kernels"] = head_kernels(a.batch, 50)
    net = pkg.Darknet(cfgs.yolov3_cfg(), dict(bench.TRAIN_HYP), arc="default")
    helpers.init_darknet_weights(net, seed=1)
    net.nc, net.hyp = 1, dict(bench.TRAIN_HYP)
    net = net.cuda().train()
    pg_w = [p for n, p in net.named_parameters() if "Conv2d.weight" in n]
    pg_o = [p for n, p in net.named_parameters() if "Conv2d.weight" not in n]
    opt = torch.optim.SGD([{"params": pg_o}, {"params": pg_w, "weight_decay": 4.569e-4}], lr=1e-4, momentum=0.97,
                          nesterov=True, fused=True)
    x = torch.rand(a.batch, 3, 608, 608, generator=torch.Generator().manual_seed(0)).cuda()
    tg = bench.make_targets(a.batch, 100).cuda()
    ms = masks(net)

    def step():
        opt.zero_grad(set_to_none=True)
        loss, _ = compute_loss(net(x), tg.clone(), net, net.hyp)
        loss.backward()
        opt.step()

    rows = []
    for graph in (False, True):
        net.use_cuda_graph = graph
        for r in range(a.rounds):
            row = {"cuda_graph": graph, "round": r}
            for name, mk in ms.items():
                for p, t in zip(net.parameters(), mk):
                    p.requires_grad_(t)
                step()
                step()               # graphs: the eager + capture step, then the first replay
                row[name + "_ms"] = event_ms(step, a.steps)
            for p in net.parameters():
                p.requires_grad_(True)
            # what a step cannot go below: the forward and the loss, no backward
            row["fwd_loss_ms"] = event_ms(lambda: compute_loss(net(x), tg.clone(), net, net.hyp), a.steps)
            rows.append(row)
            print(json.dumps(row), flush=True)
    res["step"] = rows
    res["peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "frozen_step_times.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "head_kernels"}), flush=True)


if __name__ == "__main__":
    main()
