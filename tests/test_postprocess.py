"""Detection post-processing (SURVEY section 8f rank 2): the CPU oracle against torchvision.ops.batched_nms (the
reference's own NMS, installed in this image), and the CUDA kernel against the oracle -- bit exact: same kept anchors in
the same order, identical output rows."""
import numpy as np
import pytest
import torch

from oracle.postprocess_oracle import nms_greedy, postprocess_oracle


def synth_pred(b, a, nc, seed, clusters=40, spread=12.0, obj_hi=0.9):
    """Eval-style head output: boxes clustered around a few centres (so that NMS has work), sigmoid-like scores."""
    g = torch.Generator().manual_seed(seed)
    ctr = torch.rand(b, clusters, 2, generator=g) * torch.tensor([960.0, 600.0])
    which = torch.randint(0, clusters, (b, a), generator=g)
    xy = torch.gather(ctr, 1, which[..., None].expand(-1, -1, 2)) + torch.randn(b, a, 2, generator=g) * spread
    wh = torch.rand(b, a, 2, generator=g) * 80 + 20
    obj = torch.rand(b, a, 1, generator=g) * obj_hi
    cls = torch.rand(b, a, nc, generator=g)
    return torch.cat([xy, wh, obj, cls], 2).float().contiguous()


@pytest.mark.parametrize("seed,thr", [(0, 0.65), (1, 0.45), (2, 0.3)])
def test_oracle_nms_matches_torchvision(seed, thr):
    tv = pytest.importorskip("torchvision")
    p = synth_pred(1, 3000, 8, seed)[0]
    xyxy = torch.stack([p[:, 0] - p[:, 2] / 2, p[:, 1] - p[:, 3] / 2, p[:, 0] + p[:, 2] / 2, p[:, 1] + p[:, 3] / 2], 1)
    conf, cls = torch.max(p[:, 5:], 1)
    score = p[:, 4] * conf
    # per-class torchvision.ops.nms = the definition of batched_nms (its coordinate-offset shortcut is an implementation detail)
    want = []
    for c in cls.unique():
        m = (cls == c).nonzero().flatten()
        want.append(m[tv.ops.nms(xyxy[m], score[m], thr)])
    want = torch.cat(want)
    want = want[torch.argsort(score[want], descending=True, stable=True)]
    got = nms_greedy(xyxy.numpy(), score.numpy(), cls.numpy(), thr)
    assert got.tolist() == want.tolist()
    # and batched_nms itself keeps the same set
    b = tv.ops.batched_nms(xyxy, score, cls, thr)
    assert sorted(b.tolist()) == sorted(got.tolist())


def test_oracle_postprocess_shapes():
    pred = synth_pred(3, 500, 8, 5)
    pred[1, :, 4] = 0.0                               # image with nothing above the threshold
    out = postprocess_oracle(pred, 8, conf_thre=0.3, nms_thre=0.65)
    assert out[1] is None and out[0].shape[1] == 7 and out[2].shape[1] == 7
    s = out[0][:, 4] * out[0][:, 5]
    assert (s[:-1] >= s[1:]).all() and (s >= 0.3).all()


@pytest.mark.gpu
@pytest.mark.parametrize("b,a,conf,thr,agn", [(2, 11850, 0.01, 0.65, False), (3, 1000, 0.3, 0.45, False),
                                              (1, 4096, 0.05, 0.5, True), (2, 777, 0.95, 0.65, False)])
def test_cuda_postprocess_matches_oracle(b, a, conf, thr, agn):
    from streamyolo_b200.postprocess import postprocess
    pred = synth_pred(b, a, 8, 7 + a)
    if a == 777:
        pred[0, :, 4] = 0.0
    want = postprocess_oracle(pred, 8, conf, thr, agn)
    got = postprocess(pred.cuda(), 8, conf, thr, agn)
    torch.cuda.synchronize()
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if w is None:
            assert g is None
            continue
        assert g is not None and tuple(g.shape) == tuple(w.shape), (None if g is None else g.shape, w.shape)
        assert torch.equal(g.cpu(), w), f"max diff {(g.cpu() - w).abs().max().item()}"


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_oracle_postprocess_matches_torchvision_golden(seed):
    """The committed fixtures (oracle/make_nms_golden.py, generated with torchvision's per-class NMS on the CPU: batched_nms's
    vanilla path) pin nms_greedy without needing torchvision at test time: same kept anchors, same order, rows assembled
    like yolox.utils.postprocess."""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", f"nms_{seed}.npz"))
    pred = torch.from_numpy(g["pred"])[None]
    out = postprocess_oracle(pred, 8, float(g["conf"]), float(g["thr"]), nms=nms_greedy)[0]
    keep = torch.from_numpy(g["keep"])
    p = pred[0]
    want = torch.cat([torch.stack([p[keep, 0] - p[keep, 2] / 2, p[keep, 1] - p[keep, 3] / 2, p[keep, 0] + p[keep, 2] / 2,
                                   p[keep, 1] + p[keep, 3] / 2], 1), p[keep, 4:5],
                      torch.max(p[keep, 5:], 1)[0][:, None], torch.max(p[keep, 5:], 1)[1][:, None].float()], 1)
    assert out.shape == want.shape and torch.equal(out, want)
