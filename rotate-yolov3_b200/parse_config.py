"""Darknet .cfg / hyp parsing with the reference's semantics (utils/parse_config.py:6-59, utils/utils.py:33-47),
re-implemented.  Differences, both additive:
  * the bare ``areas / ratios / angles`` anchor line of cfg/yolov3.cfg (no ``ara`` token), which makes the
    reference raise (SURVEY.md D3), is accepted and means the same as the ``ara`` grammar;
  * ``parse_model_cfg`` also accepts the cfg TEXT instead of a path (anything containing a newline)."""
import math
import os

import numpy as np


def cfg2anchors(val):
    """anchor spec -> ndarray [n, 3] of (w_px, h_px, theta_rad).

    'ara a1,a2,.. / r1,r2,.. / t1,t2,..': for area, for ratio, for angle(deg): w = sqrt(area*ratio), h = sqrt(area/ratio)
    (reference loop nest utils/parse_config.py:14-21, so index = area_i*nr*nt + ratio_i*nt + angle_i); otherwise the
    value is the path of a k-means txt with one (w, h) per line, expanded with the 12 angles (-6..5)*pi/12 (:25-31)."""
    v = val.strip()
    if "ara" in v:
        v = v[v.index("ara") + 3:]
    if "/" in v and not os.path.exists(v.strip()):
        parts = [p for p in v.split("/") if len(p.strip()) != 0]
        if len(parts) != 3:
            raise ValueError("anchor line must be 'areas / ratios / angles': %r" % val)
        areas, ratios, angles = ([float(t) for t in p.split(",") if t.strip()] for p in parts)
        out = []
        for area in areas:
            for ratio in ratios:
                for angle in angles:
                    out.append([math.sqrt(area * ratio), math.sqrt(area / ratio), angle * math.pi / 180])
        return np.array(out)
    wh = np.atleast_2d(np.loadtxt(v.strip()))
    angle = np.arange(-6, 6) * math.pi / 12
    return np.concatenate([np.column_stack((np.repeat(r[None, :], len(angle), 0), angle)) for r in wh], 0)


def parse_model_cfg(path):
    """cfg file (or text) -> list of dicts, first = [net]; values are strings except 'anchors' (ndarray);
    'convolutional' blocks get batch_normalize=0 pre-populated (reference :49-50)."""
    text = path if "\n" in path else open(path, "r").read()
    mdefs = []
    for raw in text.split("\n"):
        line = raw.strip()
        if not line or line.startswith("#"):
            continue
        if line.startswith("["):
            mdefs.append({"type": line[1:-1].rstrip()})
            if mdefs[-1]["type"] == "convolutional":
                mdefs[-1]["batch_normalize"] = 0
        else:
            key, val = line.split("=", 1)
            key = key.rstrip()
            mdefs[-1][key] = cfg2anchors(val) if "anchors" in key else val.strip()
    return mdefs


def dilation(mdef):
    """(dh, dw) of a [d-convolutional] block: the value stays the string '(a,b)' in the parsed cfg and is read as
    (int(s[1]), int(s[3])) (reference model/models.py:263)"""
    s = mdef["dilation"]
    return int(s[1]), int(s[3])


def hyp_parse(path):
    """'key: value  # comment' lines -> dict of floats (reference utils/utils.py:33-47; expressions such as
    '3.1415926/12' are evaluated arithmetically)."""
    hyp = {}
    text = path if "\n" in path else open(path, "r").read()
    for raw in text.split("\n"):
        line = raw.split("#")[0].strip()
        if not line or ":" not in line:
            continue
        k, v = line.split(":", 1)
        v = v.strip()
        try:
            hyp[k.strip()] = float(v)
        except ValueError:
            hyp[k.strip()] = float(eval(v, {"__builtins__": {}}, {}))  # noqa: S307  (arithmetic only)
    return hyp
