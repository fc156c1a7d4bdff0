"""The device NMS (nms_kernel, sy_postprocess_nms) against torchvision's batched_nms as the reference runs it: on CUDA
tensors, where torchvision 0.26 shifts every box by class * (boxes.max() + 1) and runs one class-agnostic nms whose IoU
fuses the later box's area into the sum (oracle/postprocess_oracle.py: nms_reference).

CPU (no GPU needed):
  * fma_f32 rounds once (a float64 sum on an fp32 midpoint is redone exactly);
  * with fma=False the oracle keeps what torchvision's CPU _batched_nms_coordinate_trick and nms keep, on synthetic
    predictions with 8 and 80 classes and on every case of tests/golden/nms_edges.npz;
  * the fixture holds the CUDA-path oracle's kept anchors (oracle/make_nms_edges_golden.py);
  * each fixture case changes its result when the rule it names is removed (the offsets, the FMA, the NaN propagation)
    or the per-class test is added back, and the per-class rule with rounded areas (nms_greedy, which the kernel followed
    before) fails the fixture;
  * nms_kernel compiles without spills.

GPU (H100):
  * postprocess() and ops.postprocess_nms equal a literal restatement of yolox.utils.postprocess on CUDA tensors calling
    torchvision.ops.batched_nms / nms, bit for bit (rows, order, counts): 8 images of 11 850 anchors, nc in {1, 8, 80},
    conf in {0.001, 0.01, 0.3}, nms in {0.45, 0.65}, class-aware and class-agnostic, an image without candidates; the
    fixture cases; the raw eval output of StreamYOLO-s with synthetic weights at 600x960;
  * the kernel equals the fixture (no torchvision needed)."""
import os
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle.make_nms_edges_golden import ABLATION
from oracle.postprocess_oracle import fma_f32, nms_greedy, nms_reference, postprocess_oracle, round_f32

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_postprocess import synth_pred  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nms_edges.npz")


def fixture_cases():
    g = np.load(GOLD)
    return [dict(name=str(g["names"][k]), rule=str(g["rule"][k]), nc=int(g["nc"][k]), conf=float(g["conf"][k]),
                 thr=float(g["thr"][k]), agnostic=bool(g["agnostic"][k]), pred=g[f"pred_{k}"], keep=g[f"keep_{k}"])
            for k in range(len(g["names"]))]


CASES = fixture_cases()
CASE_IDS = [c["name"] for c in CASES]


def candidates(p, nc, conf):
    """[A, 5 + nc] -> (anchor index, xyxy, score, class) of the candidates, as yolox.utils.postprocess forms them"""
    half_w, half_h = p[:, 2] / 2, p[:, 3] / 2
    xyxy = torch.stack([p[:, 0] - half_w, p[:, 1] - half_h, p[:, 0] + half_w, p[:, 1] + half_h], 1)
    cconf, cls = torch.max(p[:, 5:5 + nc], 1)
    score = p[:, 4] * cconf
    idx = (score >= conf).nonzero().flatten()
    return idx, xyxy[idx], score[idx], cls[idx]


def rows_of(p, nc, keep):
    """output rows of the kept anchors, assembled like yolox.utils.postprocess"""
    p = torch.as_tensor(p)
    keep = torch.as_tensor(keep, dtype=torch.int64)
    q = p[keep]
    cconf, cls = torch.max(q[:, 5:5 + nc], 1)
    xyxy = torch.stack([q[:, 0] - q[:, 2] / 2, q[:, 1] - q[:, 3] / 2, q[:, 0] + q[:, 2] / 2, q[:, 1] + q[:, 3] / 2], 1)
    return torch.cat([xyxy, q[:, 4:5], cconf[:, None], cls[:, None].float()], 1)


def same_bits(a, b):
    """bit equality of two fp32 tensors on the same device; a NaN equals any NaN (the device's arithmetic NaN has its
    own payload)"""
    if a.shape != b.shape:
        return False
    same = a.contiguous().view(torch.int32) == b.contiguous().view(torch.int32)
    return bool((same | (a.isnan() & b.isnan())).all())


# ================================================================================================ CPU
def test_fma_f32_rounds_once():
    """(1 + 2^-12)^2 + 2^-80: the float64 sum drops 2^-80 and lands halfway between two fp32 values, ties-to-even would
    round down; the exact value lies above the midpoint, so one rounding rounds up.  Random operands agree with Fraction."""
    a = np.float32(1 + 2.0 ** -12)
    c = np.float32(2.0 ** -80)
    assert fma_f32(a, a, c) == np.float32(1 + 2.0 ** -11 + 2.0 ** -23)
    assert fma_f32(a, a, -c) == np.float32(1 + 2.0 ** -11)
    assert np.float32(np.float64(a) * np.float64(a) + np.float64(c)) == np.float32(1 + 2.0 ** -11)   # float64 rounds twice
    rng = np.random.default_rng(0)
    x, y = (rng.standard_normal(3000).astype(np.float32) * 100 for _ in range(2))
    z = rng.standard_normal(3000).astype(np.float32) * 1e4
    want = np.array([round_f32(Fraction(float(p)) * Fraction(float(q)) + Fraction(float(r))) for p, q, r in zip(x, y, z)],
                    np.float32)
    assert np.array_equal(fma_f32(x, y, z).view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("nc,seed,conf,thr,agn", [(8, 0, 0.01, 0.65, False), (80, 1, 0.01, 0.65, False),
                                                  (80, 2, 0.3, 0.45, False), (8, 3, 0.3, 0.45, True),
                                                  (80, 4, 0.001, 0.45, True)])
def test_cpu_path_matches_torchvision(nc, seed, conf, thr, agn):
    """11 850 anchors.  batched_nms itself takes the vanilla path on the CPU above 1 000 boxes, so the trick is called by
    name; on CUDA it is what batched_nms runs."""
    pytest.importorskip("torchvision")
    from torchvision.ops import nms
    from torchvision.ops.boxes import _batched_nms_coordinate_trick
    idx, b, s, c = candidates(synth_pred(1, 11850, nc, seed)[0], nc, conf)
    want = nms(b, s, thr) if agn else _batched_nms_coordinate_trick(b, s, c.float(), thr)
    got = nms_reference(b.numpy(), s.numpy(), c.numpy(), thr, agn, fma=False)
    assert got.tolist() == want.tolist()


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_cpu_path_matches_torchvision_fixture(case):
    pytest.importorskip("torchvision")
    from torchvision.ops import nms
    from torchvision.ops.boxes import _batched_nms_coordinate_trick
    idx, b, s, c = candidates(torch.from_numpy(case["pred"]), case["nc"], case["conf"])
    want = nms(b, s, case["thr"]) if case["agnostic"] else _batched_nms_coordinate_trick(b, s, c.float(), case["thr"])
    got = nms_reference(b.numpy(), s.numpy(), c.numpy(), case["thr"], case["agnostic"], fma=False)
    assert got.tolist() == want.tolist()


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_fixture_holds_cuda_path_oracle(case):
    """the kept anchors in the fixture, and the rows postprocess_oracle (CUDA path by default) assembles from them"""
    p = torch.from_numpy(case["pred"])
    idx, b, s, c = candidates(p, case["nc"], case["conf"])
    keep = idx[nms_reference(b.numpy(), s.numpy(), c.numpy(), case["thr"], case["agnostic"])]
    assert keep.tolist() == case["keep"].tolist()
    out = postprocess_oracle(p[None], case["nc"], case["conf"], case["thr"], case["agnostic"])[0]
    assert same_bits(out, rows_of(p, case["nc"], case["keep"]))


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_fixture_case_depends_on_its_rule(case):
    idx, b, s, c = candidates(torch.from_numpy(case["pred"]), case["nc"], case["conf"])
    got = idx[nms_reference(b.numpy(), s.numpy(), c.numpy(), case["thr"], case["agnostic"], **ABLATION[case["rule"]])]
    assert got.tolist() != case["keep"].tolist()


def test_fixture_covers_the_edges():
    """every rule, 1 / 8 / 80 classes, both thresholds, class-agnostic, NaN, zero-area and negative boxes, score ties"""
    assert {c["rule"] for c in CASES} == set(ABLATION)
    assert {c["nc"] for c in CASES} == {1, 8, 80}
    assert {round(c["thr"], 2) for c in CASES} == {0.45, 0.65} and any(c["agnostic"] for c in CASES)
    boxes = np.concatenate([c["pred"][:, :4] for c in CASES])
    assert np.isnan(boxes).any() and (boxes[:, 2:4] == 0).any() and (boxes[:, 0] - boxes[:, 2] / 2 < 0).any()
    ties = [c for c in CASES if c["name"].startswith("ties")]
    assert ties and all(len(np.unique(c["pred"][:, 4])) < len(c["pred"]) for c in ties)


def test_old_per_class_rule_fails_fixture():
    """nms_greedy (per class, rounded areas: what nms_kernel computed before it followed the CUDA path) differs from the
    fixture in cases of every rule"""
    failed = set()
    for case in CASES:
        idx, b, s, c = candidates(torch.from_numpy(case["pred"]), case["nc"], case["conf"])
        with np.errstate(invalid="ignore"):
            old = idx[nms_greedy(b.numpy(), s.numpy(), c.numpy(), case["thr"], case["agnostic"])]
        if old.tolist() != case["keep"].tolist():
            failed.add(case["rule"])
    assert failed == set(ABLATION)


def test_nms_kernel_compiles_without_spills(tmp_path):
    import re
    import shutil
    import subprocess
    from streamyolo_b200 import build
    if not os.path.exists(build.NVCC) and shutil.which("nvcc") is None:
        pytest.skip("no nvcc")
    nvcc = build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")
    assert "-fmad=false" in build.SOURCES["postprocess.cu"]
    r = subprocess.run([nvcc] + build.COMMON + build.SOURCES["postprocess.cu"] + ["-c", os.path.join(build.CSRC, "postprocess.cu"),
                       "-o", str(tmp_path / "k.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout
    found = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stdout)
    hits = [f for f in found if "nms_kernel" in f[0]]
    assert hits and all(f[1:] == ("0", "0", "0") for f in hits), hits


# ================================================================================================ GPU
def live_postprocess(prediction, num_classes, conf_thre=0.7, nms_thre=0.45, class_agnostic=False):
    """[yolox 0.3.0] yolox.utils.postprocess, line for line, on the tensors it is given (CUDA here)"""
    import torchvision
    prediction = prediction.clone()
    box_corner = prediction.new(prediction.shape)
    box_corner[:, :, 0] = prediction[:, :, 0] - prediction[:, :, 2] / 2
    box_corner[:, :, 1] = prediction[:, :, 1] - prediction[:, :, 3] / 2
    box_corner[:, :, 2] = prediction[:, :, 0] + prediction[:, :, 2] / 2
    box_corner[:, :, 3] = prediction[:, :, 1] + prediction[:, :, 3] / 2
    prediction[:, :, :4] = box_corner[:, :, :4]
    output = [None for _ in range(len(prediction))]
    for i, image_pred in enumerate(prediction):
        if not image_pred.size(0):
            continue
        class_conf, class_pred = torch.max(image_pred[:, 5: 5 + num_classes], 1, keepdim=True)
        conf_mask = (image_pred[:, 4] * class_conf.squeeze() >= conf_thre).squeeze()
        detections = torch.cat((image_pred[:, :5], class_conf, class_pred.float()), 1)
        detections = detections[conf_mask]
        if not detections.size(0):
            continue
        if class_agnostic:
            nms_out_index = torchvision.ops.nms(detections[:, :4], detections[:, 4] * detections[:, 5], nms_thre)
        else:
            nms_out_index = torchvision.ops.batched_nms(detections[:, :4], detections[:, 4] * detections[:, 5],
                                                        detections[:, 6], nms_thre)
        detections = detections[nms_out_index]
        if output[i] is None:
            output[i] = detections
        else:
            output[i] = torch.cat((output[i], detections))
    return output


def check_live(pred, nc, conf, thr, agn):
    """postprocess() and ops.postprocess_nms against the live reference on the same CUDA tensor: bit for bit"""
    from streamyolo_b200 import ops
    from streamyolo_b200.postprocess import postprocess
    want = live_postprocess(pred, nc, conf, thr, agn)
    got = postprocess(pred, nc, conf, thr, agn)
    det, count = ops.postprocess_nms(pred.contiguous(), nc, conf, thr, agn)
    torch.cuda.synchronize()
    assert len(got) == len(want) == pred.shape[0]
    for i, (g, w) in enumerate(zip(got, want)):
        assert (g is None) == (w is None), i
        n = 0 if w is None else w.shape[0]
        assert int(count[i]) == n, (i, int(count[i]), n)
        if w is not None:
            assert same_bits(g, w), (i, g.shape, w.shape)
            assert same_bits(det[i, :n], w), i
    return sum(0 if w is None else w.shape[0] for w in want)


@pytest.mark.gpu
@pytest.mark.parametrize("agn", [False, True], ids=["aware", "agnostic"])
@pytest.mark.parametrize("thr", [0.45, 0.65])
@pytest.mark.parametrize("conf", [0.001, 0.01, 0.3])
@pytest.mark.parametrize("nc", [1, 8, 80])
def test_kernel_matches_live_torchvision(nc, conf, thr, agn):
    """8 images of 11 850 anchors; image 3 has no candidate"""
    pytest.importorskip("torchvision")
    pred = synth_pred(8, 11850, nc, 1000 * nc + int(conf * 1000) + int(thr * 100) + agn)
    pred[3, :, 4] = 0.0
    kept = check_live(pred.cuda(), nc, conf, thr, agn)
    assert kept > 0


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_kernel_matches_live_torchvision_fixture(case):
    pytest.importorskip("torchvision")
    check_live(torch.from_numpy(case["pred"])[None].cuda(), case["nc"], case["conf"], case["thr"], case["agnostic"])


@pytest.fixture(scope="module")
def model_output():
    """raw eval output of StreamYOLO-s with synthetic weights on 8 synthetic 600x960 frame pairs (fp32 [8, 11850, 13])"""
    from streamyolo_b200 import synth
    from test_stream import _model_s
    m = _model_s(torch.bfloat16)
    with torch.no_grad():
        out = m(synth.synth_frames(8, 600, 960, seed=5).cuda())
    return out.float().contiguous(), m.head.num_classes


@pytest.mark.gpu
@pytest.mark.parametrize("conf,thr,agn", [(0.001, 0.45, False), (0.01, 0.65, False), (0.01, 0.65, True)])
def test_kernel_matches_live_torchvision_model(model_output, conf, thr, agn):
    pytest.importorskip("torchvision")
    pred, nc = model_output
    assert tuple(pred.shape) == (8, 11850, 5 + nc)
    assert check_live(pred, nc, conf, thr, agn) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_kernel_matches_fixture(case):
    from streamyolo_b200.postprocess import postprocess
    p = torch.from_numpy(case["pred"])
    got = postprocess(p[None].cuda(), case["nc"], case["conf"], case["thr"], case["agnostic"])[0]
    torch.cuda.synchronize()
    assert got is not None and same_bits(got.cpu(), rows_of(p, case["nc"], case["keep"]))
