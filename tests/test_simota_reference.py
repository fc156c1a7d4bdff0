"""SimOTA label assignment and the Trend-Aware loss (sy_tal_loss) against the reference's get_assignments as it runs.

The reference trains with ``get_assignments`` on CUDA tensors (tal_head.py:480-712, mode "gpu"): torch.topk picks the
top-10 IoUs and each ground truth's dynamic-k anchors, ``.sum(1).int()`` gives dynamic k, torch.min(dim=0) resolves
anchors claimed twice, and F.binary_cross_entropy(...).sum(-1) is the class cost -- ATen CUDA kernels, whose roundings
(log1p(-p) in the BCE, a tree-ordered sum) and tie rules are not those of the same calls on the CPU.  ``assign_reference``
below restates get_in_boxes_info, the cost of get_assignments, dynamic_k_matching and yolox bboxes_iou(xyxy=False) as
those torch calls in the reference's order, runs unchanged on CPU and CUDA tensors, and exposes what the kernel keeps in
its workspace: the per-(GT, anchor) IoU and cost rows, each GT's dynamic k and each anchor's match count.

CPU: the restatement reproduces the assignments recorded from the unmodified reference (tests/golden/*.npz of
oracle/make_golden.py and the edge-case fixture simota_edges.npz of oracle/make_simota_edges_golden.py); each fixture case
changes its answer when the rule it names is changed (ablation); a Python mirror of the workspace layout.
GPU: the kernel's IoU and cost rows, match counts, foreground, matched ids and matched IoUs equal the restatement on CUDA
tensors bit for bit at every multi-scale grid and edge case; the kernel equals the fixture wherever the CPU and CUDA
reference agree; losses and gradients against float64 autograd; one CUDA-graph replay equals the eager calls.
"""
import functools
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.make_simota_edges_golden import LOSSES, STRIDES, anchor_grid, checksum, edge_cases, level_hw, tree_sum
from oracle.streamyolo_oracle import OracleCfg, StreamYoloOracle
from streamyolo_b200 import ops
from streamyolo_b200.train import multiscale_sizes

GOLD = os.path.join(os.path.dirname(__file__), "golden")
INF = float("inf")
U32 = 2.0 ** -24


@functools.lru_cache(maxsize=None)
def cases():
    return edge_cases()


@functools.lru_cache(maxsize=None)
def fixture():
    return dict(np.load(os.path.join(GOLD, "simota_edges.npz")))


def case_ids():
    return [c["name"] for c in cases()]


def by_name(name):
    k = case_ids().index(name)
    return k, cases()[k]


# ------------------------------------------------------------------------------------------------ the restatement
def bboxes_iou(a, b):
    """yolox bboxes_iou(a, b, xyxy=False): [Ga, Gb], no epsilon in the union"""
    tl = torch.max(a[:, None, :2] - a[:, None, 2:] / 2, b[:, :2] - b[:, 2:] / 2)
    br = torch.min(a[:, None, :2] + a[:, None, 2:] / 2, b[:, :2] + b[:, 2:] / 2)
    inside = (tl < br).type(tl.type()).prod(dim=2)
    inter = torch.prod(br - tl, 2) * inside
    return inter / (torch.prod(a[:, 2:], 1)[:, None] + torch.prod(b[:, 2:], 1) - inter)


def tree_row_sum(x):
    """fp32 sum over the last dimension in ATen's CUDA reduction order (aten_sum in head_loss.cu), on any device"""
    rows = x.detach().cpu().reshape(-1, x.shape[-1]).numpy()
    if rows.shape[0] == 0:
        return torch.zeros(x.shape[:-1], device=x.device)
    return torch.tensor([tree_sum(r) for r in rows], dtype=torch.float32).reshape(x.shape[:-1]).to(x.device)


def _pick(row, k, ties):
    """indices of the k smallest entries of row: torch.topk (ties=None) or explicitly lowest / highest index first"""
    if ties is None:
        return torch.topk(row, k=k, largest=False).indices
    if ties == "low":
        return torch.sort(row, stable=True).indices[:k]
    return row.numel() - 1 - torch.sort(row.flip(0), stable=True).indices[:k]


def assign_reference(gt, gcls, boxes, obj, cls, gx, gy, gs, nc, strict=True, ties=None, clamp=True, dk_round=False,
                     tree_sum=False, cls_tree_sum=False):
    """SimOTA for one image with the reference's operations, on whatever device the tensors live on.
    gt [G, 4] cxcywh, gcls [G], boxes [A, 4] decoded, obj [A] and cls [A, nc] logits, gx / gy / gs [A] fp32 grid.
    Ablations: strict (the in-box / in-centre tests are > 0; False: >= 0), ties (None: torch.topk / torch.min; "low",
    "high": that index first), clamp (False: a BCE term the -100 clamp decided becomes inf), dk_round (round instead of
    truncate dynamic k), tree_sum / cls_tree_sum (ATen's CUDA summation order for dynamic k / the class cost instead of
    the device's own)."""
    G, A = gt.shape[0], boxes.shape[0]
    # get_in_boxes_info
    xc = gx * gs + 0.5 * gs
    yc = gy * gs + 0.5 * gs
    l, r = gt[:, 0] - 0.5 * gt[:, 2], gt[:, 0] + 0.5 * gt[:, 2]
    t, b = gt[:, 1] - 0.5 * gt[:, 3], gt[:, 1] + 0.5 * gt[:, 3]
    d_box = torch.stack([xc[None] - l[:, None], yc[None] - t[:, None], r[:, None] - xc[None], b[:, None] - yc[None]], 2)
    rad = 2.5 * gs
    cl, cr = gt[:, 0:1] - rad[None], gt[:, 0:1] + rad[None]
    ct, cb = gt[:, 1:2] - rad[None], gt[:, 1:2] + rad[None]
    d_ctr = torch.stack([xc[None] - cl, yc[None] - ct, cr - xc[None], cb - yc[None]], 2)
    if strict:
        in_box, in_ctr = d_box.min(dim=-1).values > 0.0, d_ctr.min(dim=-1).values > 0.0
    else:
        in_box, in_ctr = d_box.min(dim=-1).values >= 0.0, d_ctr.min(dim=-1).values >= 0.0
    cand = (in_box.sum(dim=0) > 0) | (in_ctr.sum(dim=0) > 0)
    both = in_box[:, cand] & in_ctr[:, cand]
    N = int(cand.sum())
    # cost (get_assignments)
    iou = bboxes_iou(gt, boxes[cand])
    onehot = F.one_hot(gcls.to(torch.int64), nc).float().unsqueeze(1).repeat(1, N, 1)
    p = (cls[cand].float().unsqueeze(0).repeat(G, 1, 1).sigmoid_()
         * obj[cand][:, None].unsqueeze(0).repeat(G, 1, 1).sigmoid_()).sqrt_()
    terms = F.binary_cross_entropy(p, onehot, reduction="none")
    if not clamp:
        terms = torch.where(terms == 100.0, torch.full_like(terms, INF), terms)
    cost = (tree_row_sum(terms) if cls_tree_sum else terms.sum(-1)) + 3.0 * -torch.log(iou + 1e-8) + 100000.0 * (~both)
    # dynamic_k_matching
    top = torch.topk(iou, min(10, N), dim=1).values
    s = tree_row_sum(top) if tree_sum else top.sum(1)
    dyn_k = torch.clamp((torch.round(s) if dk_round else s).int(), min=1)
    M = torch.zeros_like(cost)
    for g in range(G):
        M[g][_pick(cost[g], int(dyn_k[g]), ties)] = 1.0
    count = M.sum(0)
    multi = count > 1
    if int(multi.sum()) > 0:
        sub = cost[:, multi]
        if ties is None:
            _, arg = torch.min(sub, dim=0)
        elif ties == "low":
            arg = torch.sort(sub, dim=0, stable=True).indices[0]
        else:
            arg = G - 1 - torch.sort(sub.flip(0), dim=0, stable=True).indices[0]
        M[:, multi] *= 0.0
        M[arg, multi] = 1.0
    fg_c = M.sum(0) > 0.0
    matched_c = M[:, fg_c].argmax(0)
    piou_c = (M * iou).sum(0)[fg_c]
    # back on the full anchor axis, as the kernel keeps them
    dev = boxes.device
    ci = cand.nonzero()[:, 0]
    full = lambda fill, dt: torch.full((A,), fill, dtype=dt, device=dev)
    fg = full(False, torch.bool)
    fg[ci[fg_c]] = True
    matched = full(-1, torch.int64)
    matched[ci[fg_c]] = matched_c
    pred_iou = full(0.0, torch.float32)
    pred_iou[ci[fg_c]] = piou_c
    iou_m = torch.full((G, A), -INF, device=dev)
    iou_m[:, ci] = iou
    cost_m = torch.full((G, A), INF, device=dev)
    cost_m[:, ci] = cost
    cnt = torch.zeros(A, dtype=torch.int32, device=dev)
    cnt[ci] = count.int()
    return dict(cand=cand, iou=iou_m, cost=cost_m, dyn_k=dyn_k, count=cnt, fg=fg, matched=matched, pred_iou=pred_iou)


def trend_iou(fut, cur, thr, val, le=False):
    """tal_head.py:394-403: per future GT its best IoU against the current labels, replaced by ignore_value below
    ignore_thr (le: at or below), 1 without current labels; the TAL weight is 1 / (trend IoU ** gamma + 1e-8)"""
    if cur.shape[0] == 0:
        return torch.ones(fut.shape[0], device=fut.device)
    ious, _ = torch.max(bboxes_iou(fut, cur), dim=1)
    ious[ious <= thr if le else ious < thr] = val
    return ious


class LeOracle(StreamYoloOracle):
    """the oracle with the ignore threshold applied at or below it (the rule of the TAL cases, changed)"""

    def tal_gt_iou(self, gt, sup_gt):
        if sup_gt.shape[0] == 0:
            return torch.ones(gt.shape[0])
        v = self.pairwise_iou_cxcywh(gt, sup_gt).max(1).values
        return torch.where(v <= self.cfg.ignore_thr, torch.full_like(v, self.cfg.ignore_value), v)


def oracle_f64(c, oracle_cls=StreamYoloOracle):
    """float64 losses of the oracle on case c's fp32 outputs, after total_loss.backward(): (losses, aux, d outputs,
    d origin, grid)"""
    o = oracle_cls(OracleCfg(num_classes=c["nc"], gamma=c["gamma"], ignore_thr=c["thr"], ignore_value=c["val"]), {})
    grid64 = tuple(torch.from_numpy(v).double() for v in anchor_grid(c["hw"]))
    out64 = torch.from_numpy(c["outputs"]).double().requires_grad_(True)
    org64 = torch.from_numpy(c["origin"]).double().requires_grad_(True)
    ref = o.losses(out64, org64, grid64, (torch.from_numpy(c["fut"]), torch.from_numpy(c["cur"])), return_aux=True,
                   dtype=torch.float64)
    ref["total_loss"].backward()
    return ref, out64, org64, grid64


def grad_bar(want, kappa=2.0 ** -12):
    """the gradient bar of test_tal_loss_backward_full_anchor_count: kappa * (|ref| + the rms of the column's non-zero
    entries); 2^-12 covers ~2^4 fp32 operations on coordinate differences that cost up to 2^7 of the precision"""
    nz = (want != 0).sum(0).clamp(min=1)
    rms = (want.square().sum(0) / nz).sqrt()
    return kappa * (want.abs() + rms)


def n_labels(lab):
    return int((lab.sum(1) > 0).sum())


def assign_case(c, device, b=None, **ablation):
    """assign_reference on every image of fixture case c: lists of per-image results (None for an image without labels)"""
    gx, gy, gs = (torch.from_numpy(v).to(device) for v in anchor_grid(c["hw"]))
    out = torch.from_numpy(c["outputs"]).to(device)
    fut = torch.from_numpy(c["fut"]).to(device)
    res = []
    for bi in range(out.shape[0]) if b is None else [b]:
        G = n_labels(fut[bi])
        if G == 0:
            res.append(None)
            continue
        o = out[bi]
        res.append(assign_reference(fut[bi, :G, 1:5], fut[bi, :G, 0], o[:, :4], o[:, 4], o[:, 5:], gx, gy, gs, c["nc"],
                                    **ablation))
    return res


def answer(res):
    """(image, anchor, matched GT, matched IoU) of every foreground anchor, like the fixture stores them"""
    img, anc, gt, iou = [], [], [], []
    for bi, r in enumerate(res):
        if r is None:
            continue
        a = r["fg"].nonzero()[:, 0].cpu()
        img.append(np.full(len(a), bi, np.int32))
        anc.append(a.numpy().astype(np.int32))
        gt.append(r["matched"].cpu()[a].numpy().astype(np.int32))
        iou.append(r["pred_iou"].cpu()[a].numpy().astype(np.float32))
    cat = lambda v, dt: np.concatenate(v) if v else np.zeros(0, dt)
    return cat(img, np.int32), cat(anc, np.int32), cat(gt, np.int32), cat(iou, np.float32)


def fixture_answer(k):
    f = fixture()
    return f[f"fg_image_{k}"], f[f"fg_anchor_{k}"], f[f"fg_gt_{k}"], f[f"fg_iou_{k}"]


def same_answer(x, y):
    return all(np.array_equal(a, b) for a, b in zip(x, y))


# ------------------------------------------------------------------------------------------------ workspace mirror
def carve(B, A, L, NC):
    """Python mirror of carve() in head_loss.cu: name -> (byte offset, dtype, shape), and the total size"""
    lay, off = {}, 0
    nblk = -(-A // 256) * B
    for name, dt, shape in (("ngt", torch.int32, (B,)), ("nsup", torch.int32, (B,)), ("tal", torch.float32, (B, L)),
                            ("cand", torch.int32, (B, A)), ("clsterm", torch.float32, (B, A, 2 * NC)),
                            ("iou", torch.float32, (B, L, A)), ("cost", torch.float32, (B, L, A)),
                            ("cnt", torch.int32, (B, A)), ("match", torch.int32, (B, A)),
                            ("part", torch.float64, (nblk, 8)), ("mres", torch.int32, (B, A)),
                            ("piou", torch.float32, (B, A)), ("tot", torch.float64, (8,))):
        lay[name] = (off, dt, shape)
        off = (off + int(np.prod(shape)) * torch.empty(0, dtype=dt).element_size() + 255) & ~255
    return lay, off


def ws_view(ws, lay, name):
    off, dt, shape = lay[name]
    n = int(np.prod(shape)) * torch.empty(0, dtype=dt).element_size()
    return ws[off:off + n].view(dt).reshape(shape)


@pytest.mark.parametrize("b,a,l,nc", [(1, 1, 1, 1), (2, 8150, 50, 8), (16, 11850, 120, 8), (3, 15820, 50, 80),
                                      (5, 257, 7, 3), (8, 11850, 50, 27)])
def test_workspace_mirror_matches_library(b, a, l, nc):
    assert carve(b, a, l, nc)[1] == ops.tal_loss_workspace_bytes(b, a, l, nc)


# ------------------------------------------------------------------------------------------------ CPU: pinned to the reference
def test_fixture_inputs_unchanged():
    f = fixture()
    assert f["names"].tolist() == case_ids()
    assert f["checksum"].tolist() == [checksum(c) for c in cases()]
    assert f["rule"].tolist() == [c["rule"] for c in cases()]


def test_level_grids_are_the_forward_grids():
    """level_hw (ops.conv_out_hw down the stride chain) at every multi-scale size, and at the two extremes the grid a
    model forward produces"""
    sizes = multiscale_sizes()
    grids = [c for c in cases() if c["name"].startswith("grid_")]
    assert [c["name"] for c in grids] == [f"grid_{h}x{w}" for h, w in sizes]
    assert [c["hw"] for c in grids] == [level_hw(h, w) for h, w in sizes]
    assert level_hw(496, 800) == [(62, 100), (31, 50), (16, 25)]
    from streamyolo_b200 import synth
    from oracle.streamyolo_oracle import model_shapes
    cfg = OracleCfg(depth=0.33, width=0.125)
    o = StreamYoloOracle(cfg, synth.synth_state_dict(model_shapes(0.33, 0.125)))
    o.training = False
    for h, w in (min(sizes), max(sizes)):
        with torch.no_grad():
            o.forward(synth.synth_frames(1, h, w))
        assert [tuple(x) for x in o.hw] == level_hw(h, w), (h, w)


@pytest.mark.parametrize("name", ["tiny_120x160", "tiny_empty_96x160", "s_600x960"])
def test_restatement_reproduces_golden_assignment(name):
    """on the oracle's head outputs for the golden inputs, the restatement gives the reference's foreground anchors and
    matched GTs exactly (the IoUs within the oracle forward's own distance from the reference forward)"""
    from oracle.make_golden import CASES
    from oracle.streamyolo_oracle import model_shapes
    from streamyolo_b200 import synth
    c = CASES[name]
    g = np.load(os.path.join(GOLD, name + ".npz"))
    cfg = OracleCfg(depth=c["depth"], width=c["width"], gamma=c["gamma"], ignore_thr=c["thr"], ignore_value=c["val"])
    o = StreamYoloOracle(cfg, synth.synth_state_dict(model_shapes(c["depth"], c["width"])))
    fut, _ = synth.synth_labels(c["B"], c["H"], c["W"], empty_image=c["empty"])
    with torch.no_grad():
        outputs, _, _ = o.flatten_decode(o.head_levels(o.backbone_off(synth.synth_frames(c["B"], c["H"], c["W"]))), False)
    case = dict(hw=[tuple(x) for x in o.hw], outputs=outputs.numpy(), fut=fut.numpy(), nc=8)
    img, anc, gt, iou = answer(assign_case(case, "cpu"))
    assert np.array_equal(img, g["fg_image"]) and np.array_equal(anc, g["fg_anchor"])
    assert np.array_equal(gt, g["fg_gt"])
    np.testing.assert_allclose(iou, g["fg_iou"], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("name", case_ids())
def test_restatement_reproduces_fixture(name):
    """on the fixture's own inputs the CPU restatement is the reference bit for bit: foreground, matched GTs, IoUs"""
    k, c = by_name(name)
    got = answer(assign_case(c, "cpu"))
    want = fixture_answer(k)
    assert same_answer(got, want), name
    if c["rule"] == "sum_order":                       # the boundary: the CPU's order gives the recorded dynamic k
        f = fixture()
        assert int(f[f"dk_cpu_{k}"]) != int(f[f"dk_cuda_{k}"])
        r = assign_case(c, "cpu", b=0)[0]
        assert int(r["dyn_k"][0]) == max(1, int(f[f"dk_cpu_{k}"]))
        assert int(assign_case(c, "cpu", b=0, tree_sum=True)[0]["dyn_k"][0]) == max(1, int(f[f"dk_cuda_{k}"]))


# The fixture cases where the CPU's torch.topk does not take the lowest anchor index among equal costs (the oracle's
# rule, and the rule of ATen's CUDA topk): the CPU reference's answer there depends on its partial sort.
ORACLE_DIFFERS = {"saturated"}


@pytest.mark.parametrize("name", case_ids())
def test_restatement_vs_oracle_assign(name):
    k, c = by_name(name)
    o = StreamYoloOracle(OracleCfg(num_classes=c["nc"]), {})
    grid = tuple(torch.from_numpy(v) for v in anchor_grid(c["hw"]))
    out = torch.from_numpy(c["outputs"])
    fut = torch.from_numpy(c["fut"])
    agree = agree_low = True
    for bi, (r, r_low) in enumerate(zip(assign_case(c, "cpu"), assign_case(c, "cpu", ties="low"))):
        if r is None:
            continue
        G = n_labels(fut[bi])
        fg, m, pi = o.assign(fut[bi, :G, 1:5], fut[bi, :G, 0], out[bi, :, :4], out[bi, :, 4], out[bi, :, 5:], grid)
        agree &= torch.equal(fg, r["fg"]) and torch.equal(m, r["matched"])
        agree_low &= torch.equal(fg, r_low["fg"]) and torch.equal(m, r_low["matched"])
    assert agree == (name not in ORACLE_DIFFERS), name
    assert agree_low, f"{name}: the oracle differs from the reference with lowest-index ties"


ABLATIONS = {">": dict(strict=False), "ties": dict(ties="high"), "clamp": dict(clamp=False),
             "trunc": dict(dk_round=True), "sum_order": dict(tree_sum=True)}


@pytest.mark.parametrize("name", case_ids())
def test_ablation_changes_the_answer(name):
    """changing the rule a case names changes the reference's answer on it"""
    k, c = by_name(name)
    rule = c["rule"]
    if rule == "ignore_thr":
        # the loss values do not depend on the TAL weights (normalised by their own sum, tal_head.py:432-444); the
        # gradient does.  The reference's d total_loss / d box (recorded in fp32) is the float64 gradient of the TAL
        # rule with <, within the gradient bar widened for the fp32 reference, and not that of the rule with <=
        fut, cur = torch.from_numpy(c["fut"][0]), torch.from_numpy(c["cur"][0])
        assert float(bboxes_iou(fut[:1, 1:5], cur[:1, 1:5])[0, 0]) == np.float32(c["thr"])
        f = fixture()
        bi, ai = torch.from_numpy(f[f"fg_image_{k}"]).long(), torch.from_numpy(f[f"fg_anchor_{k}"]).long()
        want = torch.from_numpy(f[f"grad_box_{k}"]).double()
        for cls, ok in ((StreamYoloOracle, True), (LeOracle, False)):
            ref, out64, _, _ = oracle_f64(c, cls)
            assert torch.equal(ref["aux"]["fg"].nonzero(), torch.stack([bi, ai], 1))
            got = out64.grad[bi, ai, 0:4]
            within = bool(((got - want).abs() <= grad_bar(want, 2.0 ** -11)).all())
            assert within == ok, f"{name}: {cls.__name__} {'misses' if ok else 'reproduces'} the reference's gradient"
        return
    got = answer(assign_case(c, "cpu", **ABLATIONS[rule]))
    assert not same_answer(got, fixture_answer(k)), f"{name}: the rule {rule!r} decides nothing here"


def test_cpu_cuda_differences_have_their_causes():
    """the causes named in CUDA_DIFFERS, shown on the CPU: with ATen's CUDA order for the class cost, crowd and
    classes_c8 change answer while lowest-index ties leave them alone; saturated changes with lowest-index ties;
    dk_sum_order with ATen's CUDA order for dynamic k"""
    for name, ablation in (("crowd", dict(cls_tree_sum=True)), ("classes_c8", dict(cls_tree_sum=True)),
                           ("saturated", dict(ties="low")), ("dk_sum_order", dict(tree_sum=True))):
        k, c = by_name(name)
        want = fixture_answer(k)
        assert not same_answer(answer(assign_case(c, "cpu", **ablation)), want), name
        if name in ("crowd", "classes_c8"):
            assert same_answer(answer(assign_case(c, "cpu", ties="low")), want), name


# ------------------------------------------------------------------------------------------------ GPU
DEV = "cuda"


def run_kernel(c, use_l1=True):
    B, A, NO = c["outputs"].shape
    L, nc = c["fut"].shape[1], c["nc"]
    lay, nbytes = carve(B, A, L, nc)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    loss = torch.empty(6, device=DEV)
    fg = torch.empty((B, A), dtype=torch.int32, device=DEV)
    mt = torch.empty((B, A), dtype=torch.int32, device=DEV)
    pi = torch.empty((B, A), device=DEV)
    t = dict(outputs=torch.from_numpy(c["outputs"]).to(DEV), origin=torch.from_numpy(c["origin"]).to(DEV),
             fut=torch.from_numpy(c["fut"]).to(DEV), cur=torch.from_numpy(c["cur"]).to(DEV))
    ops.tal_loss(t["outputs"], t["origin"], t["fut"], t["cur"], c["hw"], STRIDES, c["gamma"], c["thr"], c["val"], use_l1,
                 ws, loss, fg, mt, pi)
    torch.cuda.synchronize()
    return dict(ws=ws, lay=lay, loss=loss, fg=fg, matched=mt, pred_iou=pi, t=t)


def kernel_answer(k):
    fg = k["fg"].cpu().bool()
    bi, ai = fg.nonzero(as_tuple=True)
    return (bi.numpy().astype(np.int32), ai.numpy().astype(np.int32), k["matched"].cpu()[bi, ai].numpy().astype(np.int32),
            k["pred_iou"].cpu()[bi, ai].numpy().astype(np.float32))


def first_diff(got, want):
    bad = (got != want) & ~(torch.isnan(got) & torch.isnan(want)) if got.is_floating_point() else got != want
    i = bad.nonzero()
    return f"{int(bad.sum())} entries, first at {tuple(i[0].tolist())}: {got[tuple(i[0])].item()!r} vs {want[tuple(i[0])].item()!r}"


@pytest.mark.gpu
@pytest.mark.parametrize("name", case_ids())
def test_kernel_intermediates_equal_cuda_reference(name):
    """IoU and cost rows, match counts, foreground, matched ids and matched IoUs of sy_tal_loss equal the restatement on
    CUDA tensors bit for bit"""
    _, c = by_name(name)
    k = run_kernel(c)
    iou_w, cost_w = ws_view(k["ws"], k["lay"], "iou"), ws_view(k["ws"], k["lay"], "cost")
    cnt_w, match_w = ws_view(k["ws"], k["lay"], "cnt"), ws_view(k["ws"], k["lay"], "match")
    ngt = ws_view(k["ws"], k["lay"], "ngt").cpu()
    tal_w = ws_view(k["ws"], k["lay"], "tal")
    fut, cur = k["t"]["fut"], k["t"]["cur"]
    for bi in range(fut.shape[0]):                             # trend IoU per future GT (tal_head.py:394-403)
        G, GS = n_labels(fut[bi]), n_labels(cur[bi])
        want = trend_iou(fut[bi, :G, 1:5], cur[bi, :GS, 1:5], c["thr"], c["val"])
        assert torch.equal(tal_w[bi, :G], want), f"{name} image {bi}: trend IoUs differ: {first_diff(tal_w[bi, :G], want)}"
    for bi, r in enumerate(assign_case(c, DEV)):
        G = 0 if r is None else r["iou"].shape[0]
        assert int(ngt[bi]) == G
        if r is None:
            assert int(k["fg"][bi].sum()) == 0
            continue
        where = f"{name} image {bi}"
        assert torch.equal(iou_w[bi, :G], r["iou"]), f"{where}: IoU rows differ: {first_diff(iou_w[bi, :G], r['iou'])}"
        assert torch.equal(cost_w[bi, :G], r["cost"]), f"{where}: cost rows differ: {first_diff(cost_w[bi, :G], r['cost'])}"
        assert torch.equal(cnt_w[bi], r["count"]), f"{where}: match counts differ: {first_diff(cnt_w[bi], r['count'])}"
        assert int(cnt_w[bi].sum()) == int(r["dyn_k"].sum()), f"{where}: dynamic k differs"
        assert torch.equal(k["fg"][bi].bool(), r["fg"]), f"{where}: foreground differs"
        assert torch.equal(k["matched"][bi].long(), r["matched"]), f"{where}: matched GT ids differ"
        assert torch.equal(k["pred_iou"][bi], r["pred_iou"]), f"{where}: matched IoUs differ"
        single = cnt_w[bi] == 1                                   # an anchor one GT chose: the kernel's match is that GT
        assert torch.equal(match_w[bi][single].long(), r["matched"][single]), f"{where}: single matches differ"


# The fixture cases where the reference's answer on CUDA tensors differs from its answer on the CPU.  The kernel follows
# CUDA there: that is the reference as it trains.
#   crowd, classes_c8   the class cost: the CPU and ATen's CUDA kernel add the eight BCE terms in different orders, and
#                       the last-bit difference reorders near-equal costs (the tie rules agree here)
#   saturated           exact cost ties between saturated anchors: ATen's CUDA topk takes the lowest anchor index, the
#                       CPU's partial sort does not
#   dk_sum_order        the ten IoUs sum to different integers in the CPU's and in ATen's CUDA order
# test_cpu_cuda_differences_have_their_causes shows each cause on the CPU.
CUDA_DIFFERS = {"crowd", "classes_c8", "saturated", "dk_sum_order"}


@pytest.mark.gpu
@pytest.mark.parametrize("name", case_ids())
def test_kernel_equals_fixture(name):
    k_, c = by_name(name)
    kern = kernel_answer(run_kernel(c))
    cuda_ref = answer(assign_case(c, DEV))
    assert same_answer(kern, cuda_ref), f"{name}: the kernel differs from the CUDA reference"
    cpu_agrees = same_answer(cuda_ref, fixture_answer(k_))
    assert cpu_agrees == (name not in CUDA_DIFFERS), f"{name}: CPU and CUDA reference {'agree' if cpu_agrees else 'differ'}"


def loss_bars(ref, nfg):
    """bars for the six losses: geometric terms (IoU, L1) carry ~2^4 fp32 operations on coordinate differences that cost
    up to 2^7 of the relative precision (test_tal_loss_backward_full_anchor_count): 2^-12 relative; the BCE terms a few
    fp32 roundings each, summed in double: 2^-24 * 2^4; num_fg / num_gts: one fp32 rounding"""
    r = np.abs(ref)
    b = np.array([0.0, 2.0 ** -12 * r[1], 2.0 ** -20 * r[2], 2.0 ** -20 * r[3], 2.0 ** -12 * r[4], U32 * r[5]])
    b[0] = b[1:5].sum() + U32 * r[0]
    return b + 1e-300


GRIDS = [n for n in case_ids() if n.startswith("grid_")]
TAL = [c["name"] for c in cases() if c["rule"] == "ignore_thr"]


def kernel_backward(k, c):
    B, A, NO = c["outputs"].shape
    g_out = torch.full((B, A, NO), float("nan"), device=DEV)
    g_org = torch.full((B, A, 4), float("nan"), device=DEV)
    g_raw = torch.full((B, A, NO), float("nan"), device=DEV)
    t = k["t"]
    ops.tal_loss_backward(t["outputs"], t["origin"], t["fut"], c["hw"], STRIDES, c["gamma"], True, k["ws"], 1.0,
                          grad_outputs=g_out, grad_origin=g_org, grad_raw=g_raw)
    torch.cuda.synchronize()
    return g_out, g_org, g_raw


@pytest.mark.gpu
@pytest.mark.parametrize("name", GRIDS + TAL)
def test_grid_loss_and_gradients_vs_float64(name):
    """at every multi-scale grid and on the TAL cases (trend IoU equal to ignore_thr, future labels without current ones
    and the reverse, gamma 1.5): the six losses and the three gradients of sy_tal_loss_backward against float64 autograd
    through the oracle's loss on the same fp32 head outputs (same assignment, checked first).  The TAL weights reach only
    the gradients"""
    _, c = by_name(name)
    k = run_kernel(c)
    ref, out64, org64, grid64 = oracle_f64(c)
    aux = ref["aux"]
    assert torch.equal(k["fg"].cpu().bool(), aux["fg"]) and torch.equal(k["matched"].cpu().long(), aux["matched"])
    want = np.array([float(ref[n]) for n in LOSSES])
    got = k["loss"].cpu().double().numpy()
    err, bar = np.abs(got - want), loss_bars(want, int(aux["num_fg_raw"]))
    assert (err <= bar).all(), f"{name}: losses {got.tolist()} vs {want.tolist()}: err / bar {(err / bar).tolist()}"
    g_out, g_org, g_raw = kernel_backward(k, c)
    gout_ref, gorg_ref = out64.grad, org64.grad
    _, _, gs = grid64
    graw_ref = gout_ref.clone()
    graw_ref[..., 0:2] = gout_ref[..., 0:2] * gs[None, :, None] + gorg_ref[..., 0:2]
    graw_ref[..., 2:4] = gout_ref[..., 2:4] * out64.detach()[..., 2:4] + gorg_ref[..., 2:4]
    for got_g, want_g, what in ((g_out, gout_ref, "grad_outputs"), (g_org, gorg_ref, "grad_origin"),
                                (g_raw, graw_ref, "grad_raw")):
        got_g = got_g.cpu().double()
        assert bool(torch.isfinite(got_g).all()), what
        got_g, want_g = got_g.reshape(-1, want_g.shape[-1]), want_g.reshape(-1, want_g.shape[-1])
        err_g, tol = (got_g - want_g).abs(), grad_bar(want_g)
        assert bool((err_g <= tol).all()), f"{name} {what}: worst err / tol {float((err_g / tol.clamp(min=1e-300)).max()):.3g}"


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in case_ids() if n not in CUDA_DIFFERS])
def test_kernel_losses_equal_fixture(name):
    """the six losses the reference recorded on the CPU (fp32) against the kernel, where both assign alike: the kernel's
    bars (loss_bars) plus 2^-19 of each value for the reference's own fp32 sums (a cascade over up to 2^15 anchors);
    on the TAL cases also the reference's d total_loss / d box at the foreground anchors (the TAL weights)"""
    k_, c = by_name(name)
    f = fixture()
    k = run_kernel(c)
    want = f[f"loss_{k_}"]
    got = k["loss"].cpu().double().numpy()
    err, bar = np.abs(got - want), loss_bars(want, 0) + 2.0 ** -19 * np.abs(want)
    assert (err <= bar).all(), f"{name}: losses {got.tolist()} vs {want.tolist()}: err / bar {(err / bar).tolist()}"
    if f"grad_box_{k_}" in f:
        bi, ai = torch.from_numpy(f[f"fg_image_{k_}"]).long(), torch.from_numpy(f[f"fg_anchor_{k_}"]).long()
        g_out, _, _ = kernel_backward(k, c)
        got_g = g_out.cpu().double()[bi, ai, 0:4]
        want_g = torch.from_numpy(f[f"grad_box_{k_}"]).double()
        err_g, tol = (got_g - want_g).abs(), grad_bar(want_g, 2.0 ** -11)
        assert bool((err_g <= tol).all()), f"{name}: d box: worst err / tol {float((err_g / tol).max()):.3g}"


@pytest.mark.gpu
@pytest.mark.parametrize("name", GRIDS)
def test_grid_graph_replay_equals_eager(name):
    """the trainer replays tal_loss + tal_loss_backward from a CUDA graph per input size: one replay is bit-identical to
    the eager calls"""
    _, c = by_name(name)
    B, A, NO = c["outputs"].shape
    eager = run_kernel(c)
    t = eager["t"]
    g_e = torch.empty((B, A, NO), device=DEV)
    ops.tal_loss_backward(t["outputs"], t["origin"], t["fut"], c["hw"], STRIDES, c["gamma"], True, eager["ws"], 1.0,
                          grad_raw=g_e)
    torch.cuda.synchronize()
    ws = torch.zeros_like(eager["ws"])
    loss = torch.full((6,), float("nan"), device=DEV)
    fg, mt = torch.full_like(eager["fg"], -7), torch.full_like(eager["matched"], -7)
    pi, g_r = torch.full_like(eager["pred_iou"], float("nan")), torch.full((B, A, NO), float("nan"), device=DEV)
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            ops.tal_loss(t["outputs"], t["origin"], t["fut"], t["cur"], c["hw"], STRIDES, c["gamma"], c["thr"], c["val"],
                         True, ws, loss, fg, mt, pi)
            ops.tal_loss_backward(t["outputs"], t["origin"], t["fut"], c["hw"], STRIDES, c["gamma"], True, ws, 1.0,
                                  grad_raw=g_r)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(loss, eager["loss"]) and torch.equal(fg, eager["fg"]) and torch.equal(mt, eager["matched"])
    assert torch.equal(pi, eager["pred_iou"]) and torch.equal(g_r, g_e)
