#!/usr/bin/env python
"""Golden fixtures of the squeeze-excitation graphs: the REFERENCE Darknet (model/models.py, SELayer :16-31, forward
:244-298) run here on CPU in fp32, weights from helpers.init_darknet_weights (its generic branch gives fc.0 / fc.2
non-trivial values).

    darknet_se_golden.npz
      parse:<cfg>      the reference parser's blocks of cfg/HRSC+/yolov3_512_se.cfg and cfg/ICDAR/yolov3_608_se.cfg (JSON)
      eval_*           yolov3_512_se.cfg, eval, batch 1 at 512 x 512: head samples (with each head's |max|) and decoded rows
      train_*          yolov3_512_se.cfg, training, batch 2 at 160 x 128, loss = sum(p * G) / 100: head samples, loss,
                       running statistics of a few BN layers, gradient samples + full norms of ALL parameters (the 40 SE
                       weights included)
      small_*          SMALL_CFG below (an [se] right after a stride-2 conv, `from=-4` shortcuts that skip the SE, a concat
                       route onto an SE input), batch 4 at 64 x 48: eval and training head samples, gradient samples + full
                       norms of every parameter

Inputs, cotangents and every sample position are regenerated from seeds by tests/test_se_train_gpu.py (sample_idx below:
torch.randint on a seeded CPU generator); the fixture holds reference outputs only.  Not run by the test-suite
(the GPU box has no reference tree).  Re-run: python tests/golden/make_golden_se.py"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(REPO, "tests"))

CFG_512 = "cfg/HRSC+/yolov3_512_se.cfg"
CFG_608 = "cfg/ICDAR/yolov3_608_se.cfg"
ANCHORS = "ara 900, 3000, 9000 / 5.0 / -45, 45"


def _conv(f, k, s=1, bn=1, act="leaky"):
    return "[convolutional]\n%sfilters=%d\nsize=%d\nstride=%d\npad=1\nactivation=%s\n\n" % (
        "batch_normalize=1\n" if bn else "", f, k, s, act)


def _yolo(lo, hi):
    return "[yolo]\nmask = %d-%d\nanchors = %s\nclasses=1\nnum=6\n\n" % (lo, hi, ANCHORS)


def _se(c):
    return "[se]\nchannels=%d\n\n" % c


SC4 = "[shortcut]\nfrom=-4\nactivation=linear\n\n"
# 25 blocks: 0 conv, 1 conv/2, 2 se (after the stride-2 conv), 3-4 convs, 5 shortcut -> 1 (the SE's input), 6 se,
# 7-8 convs, 9 shortcut -> 5, 10 conv/2, 11 se, 12-13 convs, 14 shortcut -> 10, 15-17 head, 18 route -3, 19 conv,
# 20 upsample, 21 concat of 20 and 5 (the unscaled input of SE 6), 22-24 head
SMALL_CFG = ("[net]\nwidth=64\nheight=48\nchannels=3\n\n" + _conv(32, 3) + _conv(64, 3, 2) + _se(64) + _conv(32, 1)
             + _conv(64, 3) + SC4 + _se(64) + _conv(32, 1) + _conv(64, 3) + SC4 + _conv(128, 3, 2) + _se(128)
             + _conv(64, 1) + _conv(128, 3) + SC4 + _conv(64, 1) + _conv(21, 1, bn=0, act="linear") + _yolo(3, 5)
             + "[route]\nlayers = -3\n\n" + _conv(32, 1) + "[upsample]\nstride=2\n\n[route]\nlayers = -1, 5\n\n"
             + _conv(64, 3) + _conv(21, 1, bn=0, act="linear") + _yolo(0, 2))

TRAIN_STATS = (0, 12, 60, 100)     # BN layers whose running statistics are stored (stem, before an SE, deep, neck)
SEEDS = dict(eval_w=512, eval_x=5120, train_w=513, train_x=5130, train_g=5131, small_w=514, small_x=5140, small_g=5141)


def sample_idx(numel, n, seed):
    """positions of the stored samples; tests/test_se_train_gpu.py regenerates them from the same seeds"""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, numel, (n,), generator=g)


def jsonable(d):
    return {k: (np.asarray(v).tolist() if isinstance(v, np.ndarray) else v) for k, v in d.items()}


def text(s):
    return np.array(s.encode())


def head_samples(sav, key, p, n, seed):
    flat = p.detach().reshape(-1)
    sav[key] = flat[sample_idx(flat.numel(), n, seed)].numpy()
    sav[key + "_absmax"] = float(flat.abs().max())
    sav[key + "_shape"] = np.array(p.shape)


def grad_samples(model, n_of, seed0):
    """per parameter (named_parameters order j): n_of(name) samples at sample_idx(numel, n, seed0 + j) and the full norm"""
    samples, norms = [], []
    for j, (name, prm) in enumerate(model.named_parameters()):
        gflat = prm.grad.reshape(-1)
        samples.append(gflat[sample_idx(gflat.numel(), n_of(name), seed0 + j)].numpy())
        norms.append(float(gflat.norm()))
    return np.array(samples, dtype=object), np.array(norms)


def train_n(name):
    """gradient samples per parameter of the 512 training fixture: the SE weights' cosine needs more entries to be stable"""
    return 1024 if ".fc." in name else (128 if "BatchNorm2d" in name else 256)


def main():
    import make_golden as mg
    import helpers
    ru, rnms, rmodels, rn_stub = mg.import_reference()      # chdir(reference root): the cfgs name their anchor files relative
    from utils.parse_config import parse_model_cfg
    torch.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    sav = {"small_cfg": text(SMALL_CFG), "seeds": text(json.dumps(SEEDS))}
    for c in (CFG_512, CFG_608):
        sav["parse:" + c] = text(json.dumps([jsonable(b) for b in parse_model_cfg(c)]))

    # ---- yolov3_512_se.cfg, eval, batch 1 at 512 x 512 ----
    model = rmodels.Darknet(CFG_512, {"context_factor": 1.0}, arc="default")
    helpers.init_darknet_weights(model, seed=SEEDS["eval_w"])
    sav["n_params"] = sum(p.numel() for p in model.parameters())
    sav["state_names"] = np.array(list(model.state_dict().keys()))
    model.eval()
    x = torch.rand(1, 3, 512, 512, generator=torch.Generator().manual_seed(SEEDS["eval_x"]))
    with torch.no_grad():
        io, ps = model(x)
    for k, p in enumerate(ps):
        head_samples(sav, "eval_p%d" % k, p, 4096, 100 + k)
    sav["eval_io_rows"] = io[0, sample_idx(io.shape[1], 2000, 110)].numpy()
    sav["eval_io_shape"] = np.array(io.shape)
    print("eval:", tuple(io.shape), [sav["eval_p%d_absmax" % k] for k in range(3)])

    # ---- yolov3_512_se.cfg, training, batch 2 at 160 x 128 ----
    model = rmodels.Darknet(CFG_512, {"context_factor": 1.0}, arc="default")
    helpers.init_darknet_weights(model, seed=SEEDS["train_w"])
    model.train()
    x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(SEEDS["train_x"]))
    ps = model(x)
    g = torch.Generator().manual_seed(SEEDS["train_g"])
    gs = [torch.randn(p.shape, generator=g) for p in ps]
    loss = sum((p * gg).sum() for p, gg in zip(ps, gs)) / 100.0
    loss.backward()
    sav["train_loss"] = float(loss)
    for k, p in enumerate(ps):
        head_samples(sav, "train_p%d" % k, p, 4096, 200 + k)
    sav["train_names"] = np.array([n for n, _ in model.named_parameters()])
    sav["train_samples"], sav["train_norms"] = grad_samples(model, train_n, 1000)
    for i in TRAIN_STATS:
        bn = model.module_list[i].BatchNorm2d
        sav["train_rm%d" % i], sav["train_rv%d" % i] = bn.running_mean.numpy(), bn.running_var.numpy()
    print("train: loss %.5f, %d parameters (%d SE)" % (float(loss), len(sav["train_names"]),
                                                       sum(".fc." in n for n in sav["train_names"])))

    # ---- the small SE graph, batch 4 at 64 x 48: eval, training, every gradient ----
    with tempfile.NamedTemporaryFile("w", suffix=".cfg", delete=False) as f:
        f.write(SMALL_CFG)
        path = f.name
    mm = rmodels.Darknet(path, {"context_factor": 1.0}, arc="default")
    helpers.init_darknet_weights(mm, seed=SEEDS["small_w"])
    xm = torch.rand(4, 3, 48, 64, generator=torch.Generator().manual_seed(SEEDS["small_x"]))
    mm.eval()
    with torch.no_grad():
        _, pe = mm(xm)
    mm.train()
    pt = mm(xm)
    g = torch.Generator().manual_seed(SEEDS["small_g"])
    gm = [torch.randn(p.shape, generator=g) for p in pt]
    lm = sum((p * gg).sum() for p, gg in zip(pt, gm)) / 10.0
    lm.backward()
    sav["small_loss"] = float(lm)
    for k, (p, q) in enumerate(zip(pe, pt)):
        head_samples(sav, "small_pe%d" % k, p, 4096, 300 + k)
        head_samples(sav, "small_p%d" % k, q, 4096, 310 + k)
    sav["small_samples"], sav["small_norms"] = grad_samples(mm, lambda n: 1 if n.endswith("activation.weight") else 512, 2000)
    out = os.path.join(HERE, "darknet_se_golden.npz")
    np.savez_compressed(out, **sav)
    print("wrote", out, os.path.getsize(out))


if __name__ == "__main__":
    main()
