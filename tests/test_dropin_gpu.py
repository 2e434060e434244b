"""Drop-in demonstration (SURVEY.md 8b callers; VERDICT r1 missing #7): the reference's own inner loops -- restated here
statement by statement because /root/reference does not exist on the GPU box -- run against this package through the
reference's own import statements (rotate_yolov3_b200.dropin.install() provides ``utils.nms.r_nms`` etc.):

  * test.py:80-151   model(imgs) -> non_max_suppression -> per-prediction skew_bbox_iou matching loop
  * detect.py:204-213  model(img) -> non_max_suppression -> per-image detections
  * train.py:268-287 pred = model(imgs); loss = compute_loss(pred, targets, model, hyp); loss.backward(); optimizer.step()
"""
import math

import pytest
import torch

import helpers

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def shim():
    from rotate_yolov3_b200 import dropin
    return dropin.install()


def _model(train=False, size=(96, 64)):
    from model.models import Darknet                      # the reference's import line (test.py:8, detect.py:7)
    m = Darknet(helpers.mini_cfg(*size), {"context_factor": 1.0}, arc="default")
    helpers.init_darknet_weights(m, seed=11)
    m = m.cuda()
    return m.train() if train else m.eval()


def test_reference_eval_loop_runs_on_the_package(shim):
    from utils.nms.nms import non_max_suppression         # test.py:13
    from utils.utils import skew_bbox_iou                 # test.py:12 (from utils.utils import *)
    from utils.nms.r_nms import r_nms                     # utils/nms/nms.py:2
    from rotate_yolov3_b200.metrics import match_detections
    model = _model()
    width, height = 96, 64
    g = torch.Generator().manual_seed(3)
    imgs = torch.rand(3, 3, height, width, generator=g).cuda()
    conf_thres, nms_thres, iou_thres = 0.3, 0.5, 0.1
    with torch.no_grad():
        inf_out, train_out = model(imgs)                   # test.py:80
    assert inf_out.shape[0] == 3 and inf_out.shape[2] == 7 and len(train_out) == 2
    before = inf_out.clone()
    output = non_max_suppression(inf_out, conf_thres=conf_thres, nms_thres=nms_thres)    # test.py:87
    assert torch.allclose(inf_out[..., 5], before[..., 5] * before[..., 6])              # the in-place side effect (nms.py:35)
    # ground truth: for image 0 the two most confident detections themselves (so that matches exist)
    targets = []
    for si, pred in enumerate(output):
        if pred is not None and si == 0:
            for d in pred[:2]:
                targets.append([si, 0.0, float(d[0]) / width, float(d[1]) / height, float(d[2]) / width, float(d[3]) / height, float(d[4])])
    targets.append([1, 0.0, 0.5, 0.5, 0.3, 0.1, 0.2])
    targets = torch.tensor(targets).cuda()
    stats, seen = [], 0
    for si, pred in enumerate(output):                    # test.py:90-151
        labels = targets[targets[:, 0] == si, 1:]
        nl = len(labels)
        tcls = labels[:, 0].tolist() if nl else []
        seen += 1
        if pred is None:
            if nl:
                stats.append(([], torch.Tensor(), torch.Tensor(), tcls))
            continue
        correct = [0] * len(pred)
        if nl:
            detected = []
            tcls_tensor = labels[:, 0]
            tbox = labels[:, 1:6].clone()
            tbox[:, [0, 2]] *= width
            tbox[:, [1, 3]] *= height
            for i, (*pbox, pconf, pcls_conf, pcls) in enumerate(pred):
                if len(detected) == nl:
                    break
                if pcls.item() not in tcls:
                    continue
                m = (pcls == tcls_tensor).nonzero().view(-1)
                iou, bi = skew_bbox_iou(pbox, tbox[m]).max(0)           # test.py:146
                if iou > iou_thres and m[bi] not in detected:
                    correct[i] = 1
                    detected.append(m[bi])
            # the batched device-side matching (SURVEY 8f item 1) gives the same answer as the reference's loop
            assert match_detections(pred, tbox, tcls_tensor, iou_thres) == correct
        stats.append((correct, pred[:, 5].cpu(), pred[:, 7].cpu(), tcls))
    assert seen == 3 and len(stats) >= 1
    assert sum(stats[0][0]) == 2                           # image 0: both ground-truth boxes found by their own detections
    # the r_nms extension name resolves and behaves like the reference binding
    assert r_nms(torch.zeros(0, 6).cuda(), 0.5).device.type == "cpu"
    with pytest.raises(RuntimeError):
        r_nms(torch.zeros(4, 6), 0.5)


def test_reference_detect_loop_runs_on_the_package(shim):
    from utils.nms.nms import non_max_suppression
    model = _model()
    img = torch.rand(3, 64, 96).cuda()
    if img.ndimension() == 3:                              # detect.py:205-206
        img = img.unsqueeze(0)
    with torch.no_grad():
        pred, _ = model(img)                               # detect.py:209
    n = 0
    for i, det in enumerate(non_max_suppression(pred, 0.3, 0.5)):       # detect.py:213
        n += 1
        if det is not None and len(det):
            assert det.shape[1] == 8 and bool((det[:-1, 5] >= det[1:, 5]).all())
    assert n == 1


def test_reference_training_loop_runs_on_the_package(shim):
    from rotate_yolov3_b200.loss import compute_loss       # model/loss.py:266 (its .cuda() calls made device-agnostic)
    model = _model(train=True, size=(64, 48))
    hyp = {"giou": 0.1, "cls": 27.76, "cls_pw": 1.0, "obj": 20.35, "obj_pw": 1.0, "iou_t": 0.5, "ang_t": math.pi / 12,
           "reg": 1.0, "context_factor": 1.0}
    model.nc, model.hyp, model.arc = 1, hyp, "default"     # train.py:198-211
    pg0, pg1 = [], []
    for k, v in dict(model.named_parameters()).items():    # train.py:70-76
        (pg1 if "Conv2d.weight" in k else pg0).append(v)
    optimizer = torch.optim.SGD(pg0, lr=1e-3, momentum=0.9, nesterov=True)
    optimizer.add_param_group({"params": pg1, "weight_decay": 5e-4})
    imgs = torch.rand(4, 3, 48, 64).cuda()
    targets = torch.tensor([[0, 0, 0.5, 0.5, 0.4, 0.1, 0.3], [2, 0, 0.3, 0.6, 0.5, 0.12, -0.7]]).cuda()
    losses = []
    accumulate = 2
    for i in range(6):
        pred = model(imgs)                                 # train.py:268
        loss, loss_items = compute_loss(pred, targets.clone(), model, hyp)     # train.py:271
        assert torch.isfinite(loss).all()                  # train.py:272-274
        loss.backward()                                    # train.py:281
        if (i + 1) % accumulate == 0:                      # train.py:284-286: gradient accumulation over 2 batches
            optimizer.step()
            optimizer.zero_grad()
        losses.append(float(loss))
    assert losses[-1] < losses[0], losses


def test_gradient_accumulation_is_exact():
    """ADVICE r1 (high): gradients returned by the training plan must not alias plan-owned buffers -- two backward passes
    without zero_grad must leave exactly 2x the single-step gradient in every parameter.  Exactly, bit for bit: the
    step adds every reduction (BN sums, split-K weight gradients, loss sums) in a fixed order, so the second backward
    returns the same bits as the first, and g + g == 2 * g in floating point."""
    import rotate_yolov3_b200 as pkg
    m = pkg.Darknet(helpers.mini_cfg(64, 48), {"context_factor": 1.0})
    helpers.init_darknet_weights(m, seed=2)
    m = m.cuda().train()
    for mod in m.modules():                                # freeze the running statistics: identical forwards
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.momentum = 0.0
    x = torch.rand(2, 3, 48, 64).cuda()
    sum(p.float().pow(2).mean() for p in m(x)).backward()
    g1 = {n: p.grad.clone() for n, p in m.named_parameters()}
    sum(p.float().pow(2).mean() for p in m(x)).backward()
    for n, p in m.named_parameters():
        # an aliased gradient buffer would be wiped, then doubled; a reduction that added in arrival order would differ
        # in the last bits, which 13 layers of training-mode BN amplify to percents at the stem
        assert torch.equal(p.grad, 2 * g1[n]), n
