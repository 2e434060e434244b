"""TEST INFRASTRUCTURE: the inputs of the focal-loss golden (tests/golden/make_golden_focal.py -> loss_focal_golden.npz).
The golden stores outputs only; the generator and the tests rebuild the inputs here from loss_golden.npz (heads, targets,
hyp of tests/golden/make_golden.py section 9) and from seeds."""
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GAMMAS = (0.5, 2.0)
OBJ_PWS = (1.0, 2.0)
EXTREME = 40.0


def base_inputs():
    """heads [3 x (4, 3, ny, nx, 7)], targets [9, 7] and hyp (without fl_gamma) of loss_golden.npz"""
    g = np.load(os.path.join(GOLDEN, "loss_golden.npz"))
    hyp = {str(k): float(v) for k, v in zip(g["hyp_keys"], g["hyp_vals"])}
    return [torch.from_numpy(g["p%d" % k]).clone() for k in range(3)], torch.from_numpy(g["targets"]).clone(), hyp


def focal_hyp(hyp, gamma, obj_pw):
    h = dict(hyp)
    h["fl_gamma"], h["obj_pw"] = float(gamma), float(obj_pw)
    return h


def extreme_heads(ps, seed=61):
    """case (c): the objectness logits of every cell replaced by a seeded shuffle of an even spread over [-40, 40] with
    one cell in eight exactly 0.  At x = -40 with t = 0 the BCE loss is ~4e-18, so the focal base 1.000001 - exp(-l)
    sits at its floor 2^-20; at x = +40 with t = 0 it is 40 and the base is 1 + 2^-20."""
    gen = torch.Generator().manual_seed(seed)
    out = []
    for p in ps:
        q = p.clone()
        n = q[..., 5].numel()
        v = torch.linspace(-EXTREME, EXTREME, n)[torch.randperm(n, generator=gen)]
        v[torch.randperm(n, generator=gen)[: n // 8]] = 0.0
        q[..., 5] = v.view(q.shape[:4])
        out.append(q)
    return out


def darknet_case():
    """case (d): the Darknet-53 graph at 160 x 128 of make_golden.py section 7 (weights seed 321, x seed 11, batch 4)
    trained with the Fdefault compute_loss on the targets of loss_golden.npz, gamma 0.5"""
    x = torch.rand(4, 3, 128, 160, generator=torch.Generator().manual_seed(11))
    _, targets, hyp = base_inputs()
    return x, targets, focal_hyp(hyp, 0.5, hyp["obj_pw"])


def cases():
    """(golden tag, heads, targets, hyp) of cases (a)-(c)"""
    heads, tg, hyp0 = base_inputs()
    out = []
    for gm in GAMMAS:
        for pw in OBJ_PWS:
            out.append(("a_g%g_pw%g" % (gm, pw), heads, tg, focal_hyp(hyp0, gm, pw)))
        out.append(("b_g%g" % gm, heads, torch.zeros(0, 7), focal_hyp(hyp0, gm, hyp0["obj_pw"])))
        out.append(("c_g%g" % gm, extreme_heads(heads), tg, focal_hyp(hyp0, gm, hyp0["obj_pw"])))
    return out


def golden():
    return np.load(os.path.join(GOLDEN, "loss_focal_golden.npz"), allow_pickle=True)
