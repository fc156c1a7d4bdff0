"""Virtual ranks (train.Trainer(virtual_ranks=K), train_loop.DeviceTrainer through dropin.install(virtual_ranks=K)): K
ranks of a W x K-rank data-parallel run executed one after another in each of W processes must train as W x K processes
would (the reference's ``-d 8`` recipe, exps/train_utils/double_trainer.py:99-123, 171-175, 221-226, on fewer GPUs).

CPU: every kernel emulated (tests/emul_ops.py, exact), W processes as gloo subprocesses.  Per rank, the first step's
losses, BatchNorm buffers and EMA buffers are bit-identical to the W x K-process run; the gradient-derived state
(parameters, momentum, EMA parameters) differs only by the order in which the W x K shard gradients are summed: a
process adds shard k's walk onto the flat gradient the walks before it left (a module the walk reaches twice, the DFP
jian convs, adds its second contribution on top of the earlier ranks' sum), where gloo sums finished gradients.
GPU: the graphed step against the eager one, the accumulated gradient against K separate walks, the memory of K micro-steps
and a non-finite shard."""
import copy
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_ops  # noqa: E402
import test_cpu_backward as T  # noqa: E402
from oracle.make_golden import CASES  # noqa: E402
from streamyolo_b200 import ops, synth, train  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS = 3
PAIRS = 1           # frame pairs per rank

WORKER = r"""
import os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
import torch
import emul_ops, test_cpu_backward as T
from oracle.make_golden import CASES
from streamyolo_b200 import dist as d, synth, train


class MP:
    def setattr(self, o, n, v): setattr(o, n, v)
    def setitem(self, dct, k, v): dct[k] = v


out, K, steps, pairs = sys.argv[2], int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5])
world = int(os.environ.get("WORLD_SIZE", "1"))
rank = 0
if world > 1:
    rank, _, world = d.init("gloo")
emul_ops.install(MP(), exact=True)
c = CASES["tiny_120x160"]
n = world * K * pairs
mine = slice(rank * K * pairs, (rank + 1) * K * pairs)
model = T.build_product(c)
tr = train.Trainer(model, lr=1e-3, bucket_bytes=64 << 10, virtual_ranks=K)
res = {"loss": [], "buffers": [], "ema_buffers": []}
names = [k for k, _ in model.named_buffers()]
for s in range(steps):
    x = synth.synth_frames(n, c["H"], c["W"], seed=100 + s)
    fut, cur = synth.synth_labels(n, c["H"], c["W"], seed=1 + s)
    tr.step(x[mine], (fut[mine], cur[mine]))
    res["loss"].append([torch.stack([v.detach() for v in r.values()]) for r in tr.rank_losses()])
    sd = tr.state_dict()
    ranks = sd.get("virtual_ranks") or [{"buffers": {k: sd["model"][k] for k in names},
                                        "ema": {k: sd["ema"][k] for k in names}}]
    res["buffers"].append([{k: v.clone() for k, v in r["buffers"].items()} for r in ranks])
    res["ema_buffers"].append([{k: v.clone() for k, v in r["ema"].items()} for r in ranks])
    fs = tr.fs
    for key, t in (("param", fs.state[:fs.n_param]), ("mom", fs.mom), ("ema_param", fs.ema[:fs.n_param])):
        res.setdefault(key, []).append(t.clone())
torch.save(res, os.path.join(out, f"rank{rank}.pt"))
print("ok", rank)
"""


def _run(tmp_path, world, K, steps=STEPS):
    """W gloo processes with K virtual ranks each -> per global rank g: losses, buffers, EMA buffers (per step), and the
    gradient-derived state of process 0"""
    out = tmp_path / f"w{world}k{K}"
    out.mkdir()
    script = tmp_path / "vr_worker.py"
    script.write_text(WORKER)
    port = 29600 + (os.getpid() * 7 + 13 * world + K) % 90
    procs = []
    for r in range(world):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port), OMP_NUM_THREADS="2")
        procs.append(subprocess.Popen([sys.executable, str(script), ROOT, str(out), str(K), str(steps), str(PAIRS)],
                                      env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=900)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), "\n".join(o[-3000:] for o in outs)
    res = [torch.load(out / f"rank{r}.pt") for r in range(world)]
    flat = {key: [[row for r in res for row in r[key][s]] for s in range(steps)] for key in ("loss", "buffers", "ema_buffers")}
    flat.update({key: res[0][key] for key in ("param", "mom", "ema_param")})
    return flat


def _close(a, b, rel):
    """|a - b| <= rel * max|b| + 1e-12: the bar for state that the two runs compute from differently summed gradients"""
    return float((a - b).abs().max()) <= rel * float(b.abs().max()) + 1e-12


def _compare(got, want, ranks, addends):
    for g in range(ranks):
        assert torch.equal(got["loss"][0][g], want["loss"][0][g]), g
        for key in ("buffers", "ema_buffers"):
            for k, v in want[key][0][g].items():
                assert torch.equal(got[key][0][g][k], v), (key, g, k)
        for s in range(1, STEPS):                   # computed from parameters that differ by reassociation already
            assert _close(got["loss"][s][g], want["loss"][s][g], 1e-3), (s, g)
            for key in ("buffers", "ema_buffers"):
                for k, v in want[key][s][g].items():
                    if v.dtype.is_floating_point:
                        assert _close(got[key][s][g][k], v, 1e-3), (key, s, g, k)
                    else:
                        assert torch.equal(got[key][s][g][k], v), (key, s, g, k)
    # the first step's gradient is the same `addends` fp32 shard gradients summed in another order: a few ulps of the
    # largest element.  The later steps' gradients come from parameters that differ already, and on this random-init
    # net the difference grows about 60x per step (momentum after three steps of four ranks: 2.5e-3 of its largest
    # element), so the bar grows 200x per step.
    for key in ("param", "mom", "ema_param"):
        for s in range(STEPS):
            assert _close(got[key][s], want[key][s], 4 * addends * 2.0 ** -24 * 200 ** s), (key, s)


def test_two_virtual_ranks_match_two_gloo_ranks(tmp_path):
    """K = 2 in one process against two gloo processes, three steps."""
    _compare(_run(tmp_path, 1, 2), _run(tmp_path, 2, 1), 2, 2)


def test_four_virtual_ranks_match_four_gloo_ranks(tmp_path):
    """K = 4 in one process, and two gloo processes of K = 2, against four gloo processes."""
    want = _run(tmp_path, 4, 1)
    _compare(_run(tmp_path, 1, 4), want, 4, 4)
    _compare(_run(tmp_path, 2, 2), want, 4, 4)


def _counting(monkeypatch, calls):
    for n in emul_ops.NAMES:
        fn = getattr(ops, n)
        monkeypatch.setattr(ops, n, lambda *a, _fn=fn, _n=n, **kw: (calls.append(_n), _fn(*a, **kw))[1])


def test_one_virtual_rank_is_the_trainer_before_virtual_ranks(monkeypatch):
    """virtual_ranks=1, and a Trainer built without the argument: two steps of the tiny model make the same kernel
    entry-point calls in the same order as the Trainer before virtual ranks existed, and reach its losses and state.
    tests/golden/trainer_k1_before_virtual_ranks.json was recorded from that Trainer with this test's inputs: the call
    names of each step, the losses, fp64 sums and absolute sums of the flat state, momentum, EMA copy and gradient, and
    the state_dict keys.  The sums are compared to 1e-9 relative, so that another CPU's float kernels may differ in the
    last bits; the emulated kernels are the same on both sides."""
    import json
    with open(os.path.join(ROOT, "tests", "golden", "trainer_k1_before_virtual_ranks.json")) as fh:
        want = json.load(fh)
    emul_ops.install(monkeypatch, exact=True)
    calls = []
    _counting(monkeypatch, calls)
    c = CASES["tiny_120x160"]
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"])
    for kw in ({}, {"virtual_ranks": 1}):
        tr = train.Trainer(T.build_product(c), lr=1e-3, bucket_bytes=64 << 10, **kw)
        for i in range(2):
            del calls[:]
            got = tr.step(x, tg)
            assert calls == want["calls"][i], (kw, i)
            for k, v in want["losses"][i].items():
                assert abs(float(got[k]) - v) <= 1e-6 * abs(v), (kw, i, k)
        for name in ("state", "mom", "ema", "grad"):
            t = getattr(tr.fs, name).double()
            assert t.numel() == want[name]["numel"], name
            for key, v in (("sum", float(t.sum())), ("abs_sum", float(t.abs().sum()))):
                assert abs(v - want[name][key]) <= 1e-9 * want[name]["abs_sum"], (kw, name, key, v, want[name][key])
        assert list(tr.state_dict()) == want["state_dict_keys"]


def _tiny_k(monkeypatch, K, steps=1):
    emul_ops.install(monkeypatch, exact=True)
    c = CASES["tiny_120x160"]
    x = synth.synth_frames(K * PAIRS, c["H"], c["W"])
    tg = synth.synth_labels(K * PAIRS, c["H"], c["W"])
    model = T.build_product(c)
    tr = train.Trainer(model, lr=1e-3, virtual_ranks=K)
    for _ in range(steps):
        tr.step(x, tg)
    return c, tr, model, x, tg


def test_virtual_rank_checkpoints_and_all_reduce_norm(monkeypatch):
    """state_dict carries all K copies and resumes exactly; a different K is refused; the reference checkpoint is
    virtual rank 0's and loads into every copy; all_reduce_norm writes the mean of the K copies into every copy; a batch
    K does not divide is refused."""
    K = 2
    c, tr, model, x, tg = _tiny_k(monkeypatch, K)
    names = [n for n, _ in model.named_buffers()]
    bufs = [{n: t.clone() for n, t in r["buffers"].items()} for r in tr.state_dict()["virtual_ranks"]]
    assert not torch.equal(bufs[0][names[0]], bufs[1][names[0]])           # the two shards' statistics differ
    assert all(torch.equal(model.state_dict()[n], bufs[0][n]) for n in names)  # outside a step: rank 0's
    one = T.build_product(c)                                   # num_batches_tracked counts steps: as a one-rank step
    train.Trainer(one, lr=1e-3).step(x[:PAIRS], tuple(t[:PAIRS] for t in tg))
    counts = {n: t for n, t in one.state_dict().items() if n.endswith("num_batches_tracked")}
    assert all(torch.equal(bufs[k][n], v) for k in range(K) for n, v in counts.items())
    snap = copy.deepcopy(tr.state_dict())
    tr.step(x, tg)
    want = copy.deepcopy(tr.state_dict())
    m2 = T.build_product(c)
    t2 = train.Trainer(m2, lr=1e-3, virtual_ranks=K)
    t2.load_state_dict(snap)
    t2.step(x, tg)
    got = t2.state_dict()
    for k in range(K):
        for which in ("buffers", "ema"):
            for n, v in want["virtual_ranks"][k][which].items():
                assert torch.equal(got["virtual_ranks"][k][which][n], v), (k, which, n)
    assert torch.equal(t2.fs.state, tr.fs.state) and torch.equal(t2.fs.ema, tr.fs.ema)
    with pytest.raises(ValueError, match="virtual ranks"):
        train.Trainer(T.build_product(c), lr=1e-3, virtual_ranks=3).load_state_dict(snap)
    with pytest.raises(ValueError, match="virtual ranks"):
        train.Trainer(T.build_product(c), lr=1e-3).load_state_dict(snap)
    with pytest.raises(ValueError, match="cannot be cut"):
        tr.step(x[:1], tuple(t[:1] for t in tg))
    # reference checkpoint: rank 0's EMA weights; loading it puts its buffers into every copy
    ck = tr.reference_checkpoint(1)
    ema0 = tr.ema_state_dict(0)
    assert all(torch.equal(ck["model"][n], ema0[n]) for n in ema0)
    assert not torch.equal(tr.ema_state_dict(1)[names[0]], ema0[names[0]])
    t3 = train.Trainer(T.build_product(c), lr=1e-3, virtual_ranks=K)
    t3.load_reference_checkpoint(copy.deepcopy(ck), 5)
    for r in t3.state_dict()["virtual_ranks"]:
        for n in names:
            assert torch.equal(r["buffers"][n], ck["model"][n]), n
            assert torch.equal(r["ema"][n], ck["model"][n]), n
    # all_reduce_norm: the mean of the copies in every copy
    rb = [{n: t.clone() for n, t in r["buffers"].items()} for r in tr.state_dict()["virtual_ranks"]]
    tr.all_reduce_norm()
    after = tr.state_dict()["virtual_ranks"]
    for n in names:
        if rb[0][n].dtype.is_floating_point:
            mean = (rb[0][n] + rb[1][n]) / K
            assert torch.equal(after[0]["buffers"][n], mean) and torch.equal(after[1]["buffers"][n], mean), n
    assert torch.equal(model.state_dict()[names[0]], after[0]["buffers"][names[0]])


# ------------------------------------------------------------------------------------------------ GPU
def _graph_equals_eager_k(build, sizes, input_size, pairs, K):
    """three iterations with a size switch: the graphs of capture_sizes (K micro-steps each) against eager steps"""
    from test_multiscale_train import _Inputs, _assert_same, _snapshot
    dev = torch.device("cuda")
    seq, lrs = [sizes[0], sizes[-1], sizes[0]], [1e-4, 2e-4, 3e-4]
    inp = _Inputs(K * pairs, input_size, False, dev, sizes)
    ta = train.Trainer(build(), lr=1e-4, virtual_ranks=K)
    want = []
    for i, (s, lr) in enumerate(zip(seq, lrs)):
        inp.load(100 + i)
        x, tg = inp.eager(s)
        ta.step(x, tg, lr=lr)
        want.append([float(r["total_loss"]) for r in ta.rank_losses()])
    torch.cuda.synchronize()
    del inp
    inp = _Inputs(K * pairs, input_size, False, dev, sizes)
    tb = train.Trainer(build(), lr=1e-4, virtual_ranks=K)
    before = _snapshot(tb)
    tb.capture_sizes(sizes, inp.make_inputs, inp.prologue)
    torch.cuda.synchronize()
    _assert_same(_snapshot(tb), before, "after capture_sizes")
    got = []
    for i, (s, lr) in enumerate(zip(seq, lrs)):
        inp.load(100 + i)
        tb.replay_size(s, lr=lr)
        got.append([float(r["total_loss"]) for r in tb.rank_losses()])
    torch.cuda.synchronize()
    assert got == want, (got, want)
    assert len({v for row in got for v in row}) > K                 # the ranks' shards differ
    _assert_same(_snapshot(tb), _snapshot(ta), "after the steps")
    for a, b in zip(tb.state_dict()["virtual_ranks"], ta.state_dict()["virtual_ranks"]):
        for n, v in b["buffers"].items():
            assert torch.equal(a["buffers"][n], v), n


@pytest.mark.gpu
def test_graphed_k4_equals_eager_k4_tiny():
    from test_gpu_model import build_product
    from test_multiscale_train import TINY_SIZES
    c = CASES["tiny_120x160"]
    _graph_equals_eager_k(lambda: build_product(c["depth"], c["width"]).train(), TINY_SIZES[:3] + [(120, 192)],
                          (120, 192), 2, 4)


@pytest.mark.gpu
def test_graphed_k4_equals_eager_k4_s():
    """StreamYOLO-s at 600x960 and the largest multi-scale size, 2 pairs per virtual rank"""
    from test_gpu_parity_fwd import _build
    _graph_equals_eager_k(lambda: _build("s"), [(688, 1120), (600, 960)], (600, 960), 2, 4)


@pytest.mark.gpu
def test_accumulated_gradient_is_the_sum_of_the_shard_walks():
    """the flat gradient of one K = 4 forward_backward against the sum of four backward.forward_backward walks, each on
    its shard in a model of its own (so with copy k's buffers); every copy's statistics equal that model's bit for bit"""
    from test_gpu_model import build_product
    c = CASES["tiny_120x160"]
    K, b = 4, 2
    build = lambda: build_product(c["depth"], c["width"]).train()    # noqa: E731
    x = synth.synth_frames(K * b, 120, 192, seed=21).cuda()
    fut, cur = (t.cuda() for t in synth.synth_labels(K * b, 120, 192, seed=22))
    tr = train.Trainer(build(), lr=1e-3, virtual_ranks=K)
    tr.forward_backward(x, (fut, cur))
    torch.cuda.synchronize()
    got = tr.fs.grad.clone()
    total, absum = torch.zeros_like(got), torch.zeros_like(got)
    ranks = tr.state_dict()["virtual_ranks"]
    for k in range(K):
        m = build()
        sl = slice(k * b, (k + 1) * b)
        from streamyolo_b200.model import backward
        backward.forward_backward(m, x[sl], (fut[sl], cur[sl]))
        g = torch.zeros_like(got)
        for p, q in zip(tr.model.parameters(), m.parameters()):
            o, n = tr.fs.offset[id(p)]
            g[o:o + n] = q.grad.reshape(-1).float()
        total += g
        absum += g.abs()
        for n, v in m.state_dict().items():
            if n in ranks[k]["buffers"]:
                assert torch.equal(ranks[k]["buffers"][n], v), (k, n)
    bar = 4 * K * 2.0 ** -24 * absum
    bad = (got - total).abs() > bar
    assert not bool(bad.any()), (int(bad.sum()), float((got - total).abs().max()))


@pytest.mark.gpu
def test_memory_of_four_micro_steps_s():
    """max_memory_reserved of the K = 4 graph against K = 1 at the same per-rank batch (StreamYOLO-s, 2 pairs per rank,
    600x960): the pool holds one micro-step's activations; what K adds is the buffer copies and the larger inputs"""
    import gc
    from test_gpu_parity_fwd import _build
    dev = torch.device("cuda")
    peaks, extra = {}, {}
    for K in (1, 4):
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        x = synth.synth_frames(2 * K, 600, 960, seed=3).to(dev)
        tg = tuple(t.to(dev) for t in synth.synth_labels(2 * K, 600, 960, seed=4))
        tr = train.Trainer(_build("s"), lr=1e-4, virtual_ranks=K)
        tr.capture(x, tg)
        loss = tr.replay()["total_loss"]
        torch.cuda.synchronize()
        assert bool(torch.isfinite(loss))
        peaks[K] = torch.cuda.max_memory_reserved()
        extra[K] = 2 * 4 * (K - 1) * tr.fs.n_buf + x.numel() * 4 + sum(t.numel() * 4 for t in tg)
        del tr, x, tg
    allowed = 1.1 * peaks[1] + extra[4] - extra[1]
    print(f"\nmax_memory_reserved: K=1 {peaks[1] / 2 ** 30:.3f} GiB, K=4 {peaks[4] / 2 ** 30:.3f} GiB, ratio "
          f"{peaks[4] / peaks[1]:.3f}, extra copies + inputs {(extra[4] - extra[1]) / 2 ** 20:.1f} MiB")
    assert peaks[4] <= allowed, (peaks, allowed)


@pytest.mark.gpu
def test_nonfinite_gradient_in_one_shard_skips_the_step():
    """a NaN planted into the gradient during virtual rank 2's walk: the step leaves the parameters and momentum of the
    whole state as they were, the EMA copy (every rank's buffers included) still moves as ModelEMA.update does, and the
    skip counts once"""
    from test_gpu_model import build_product
    from streamyolo_b200.model import backward
    c = CASES["tiny_120x160"]
    K, b = 4, 2
    x = synth.synth_frames(K * b, 120, 192, seed=5).cuda()
    tg = tuple(t.cuda() for t in synth.synth_labels(K * b, 120, 192, seed=6))
    tr = train.Trainer(build_product(c["depth"], c["width"]).train(), lr=1e-3, virtual_ranks=K, skip_nonfinite=True)
    tr.step(x, tg)
    torch.cuda.synchronize()
    assert tr.skipped_steps() == 0
    state, mom, ema = tr.fs.state.clone(), tr.fs.mom.clone(), tr.fs.ema.clone()
    planted = []

    def hook(stage, r, **kw):
        if stage == "post" and tr.fs.selected == 2 and not planted:
            kw["dw"].view(-1)[0] = float("nan")
            planted.append(True)

    old, backward.DEBUG_HOOK = backward.DEBUG_HOOK, hook
    try:
        tr.step(x, tg)
    finally:
        backward.DEBUG_HOOK = old
    torch.cuda.synchronize()
    n = tr.fs.n_param
    assert planted and tr.skipped_steps() == 1
    assert torch.equal(tr.fs.state[:n], state[:n]) and torch.equal(tr.fs.mom, mom)
    assert bool(torch.isfinite(tr.fs.state[n:]).all())               # the shards' forwards ran and moved the statistics
    d = tr.ema_decay * (1 - __import__("math").exp(-tr.updates / 2000))
    want = ema.clone()
    want.mul_(d).add_((1.0 - d) * tr.fs.state)
    assert torch.allclose(tr.fs.ema, want, rtol=2 ** -22, atol=0), float((tr.fs.ema - want).abs().max())
    assert not torch.equal(tr.fs.ema, ema)


@pytest.mark.gpu
def test_device_trainer_k2_is_the_hand_wired_graphed_loop(tmp_path, monkeypatch):
    """three epochs of the drop-in loop with two virtual ranks of two pairs (host slots and graphs of four pairs, a
    random_resize size in between) == the hand-wired capture_sizes loop of a Trainer(virtual_ranks=2) fed the same
    files, labels, mirror bits, sizes and lrs: the whole flat state, momentum, EMA and every iteration's losses bit for
    bit (with all_reduce_norm after every epoch, as the drop-in runs it), and the log lines show virtual rank 0's
    losses"""
    import test_train_loop as L
    table = L.make_table(str(tmp_path / "data"), 22, "onex", hw=(240, 384), seed=1, jpeg=True, max_rows=6)
    t, exp, mod = L._gpu_loop(tmp_path, monkeypatch, "onex", table, max_epoch=3, args=L.args_for(batch_size=4),
                              run=False)
    type(t).virtual_ranks = 2
    exp.evaluator = types.SimpleNamespace(evaluate_virtual_ranks=lambda *a, **kw: (0.0, 0.0, "summary"))
    t.train()
    rec = list(L.RecordingStep.record)
    assert t.tr.virtual_ranks == 2 and t.max_iter == 6
    assert len(rec) == 18 and len({s for _, s, _, _ in rec}) == 2 and rec[0][0]["mirror"].shape[0] == 4
    base = train.Trainer

    class HandWired(base):          # the drop-in's all_reduce_norm after every epoch (averages the two ranks' statistics)
        def __init__(self, *a, **kw):
            super().__init__(*a, virtual_ranks=2, **kw)
            self.replays = 0

        def replay_size(self, size, lr=None):
            if self.replays and self.replays % t.max_iter == 0:
                self.all_reduce_norm()
            self.replays += 1
            return super().replay_size(size, lr)

    monkeypatch.setattr(train, "Trainer", HandWired)
    tr, losses = L._hand_wired("onex", rec, table, lr0=0)
    tr.all_reduce_norm()
    torch.cuda.synchronize()
    for name in ("state", "mom", "ema"):
        assert torch.equal(getattr(t.tr.fs, name), getattr(tr.fs, name)), name
    for i, ((_, _, _, got), want) in enumerate(zip(rec, losses)):
        for k in want:
            assert torch.equal(got[k], want[k]), (i, k)
    r0, r1 = (float(r["total_loss"]) for r in tr.rank_losses())
    assert r0 == float(losses[-1]["total_loss"]) and r0 != r1
    lines = [ln for ln in mod.logger.lines if ln.startswith("epoch: ")]
    assert len(lines) == 3                                      # iteration 4 of 6, every epoch
    for ln, i in zip(lines, (3, 9, 15)):
        for k in ("total_loss", "iou_loss", "l1_loss", "conf_loss", "cls_loss"):
            assert "{}: {:.1f}".format(k, float(losses[i][k])) in ln, (i, k, ln)


# ------------------------------------------------------------------------------------------------ DeviceTrainer (CPU)
def _recording_evaluator(n_val=11, batch=4):
    """a DeviceEvaluator (the drop-in subclass of the eval tests' stand-in reference evaluator) whose batch loop is
    replaced by a record of what it was asked to run: the batches and the weights the model held; its rows carry the
    dataset indices as image ids, so the scored list shows the order of the shards"""
    import test_eval_pipeline as E
    from streamyolo_b200 import evaluate
    cls = evaluate.device_evaluator(E.StandIn, "onex")
    ev = cls(E.loader(E._dataset(["a.jpg", "b.jpg", "c.jpg", "d.jpg"], "onex", n=n_val), batch), (120, 192), 0.01, 0.65, 8)
    ev.calls = []

    def rows_of(model, half):
        ev.calls.append({"batches": [list(b) for b in ev.batches],
                         "state": {k: v.detach().clone() for k, v in model.state_dict().items()}})
        idx = np.array([i for b in ev.batches for i in b], np.int64)
        return {"bbox": np.zeros((len(idx), 4), np.float32), "score": np.ones(len(idx), np.float32), "image_id": idx,
                "category_id": np.zeros(len(idx), np.int64)}, 1.0

    ev._rows_of = rows_of
    return ev


class EagerStep:
    """stand-in for train_loop.DeviceStep whose replay runs the real Trainer's step (kernels emulated) on synthetic
    pairs of the step's batch, recording every virtual rank's losses"""
    log = None

    def __init__(self, tr, table, batch, input_size, sizes, max_bytes, device):
        import test_train_loop as L
        self.fake = L.FakeStep(tr, table, batch, input_size, sizes, max_bytes, device)
        self.tr, self.batch, self.host, self.rank_rows, self.losses = tr, batch, self.fake.host, [], None
        EagerStep.log = self

    def slot_free(self, s):
        pass

    def h2d(self, s):
        self.fake.h2d(s)

    def capture(self, s):
        pass

    def replay(self, s, size, lr):
        self.fake.replays.append({"slot": self.fake.dev[s], "size": tuple(size), "lr": lr})
        k = len(self.fake.replays)
        x = synth.synth_frames(self.batch, 120, 160, seed=k)
        tg = synth.synth_labels(self.batch, 120, 160, seed=k)
        self.losses = self.tr.step(x, tg, lr=1e-3)
        self.rank_rows.append([{n: float(v) for n, v in r.items()} for r in self.tr.rank_losses()])
        self.fake.status.append(np.zeros(len(self.fake.dev[s]["lengths"]), np.int32))
        return self.losses

    def sync(self, pending):
        return self.fake.status[-pending:]

    def close(self):
        pass


def _loop(tmp_path, monkeypatch, K, world, rank, batch_size, step=None, evaluator=None):
    import test_train_loop as L
    from streamyolo_b200 import train_loop
    emul_ops.install(monkeypatch, exact=True)
    mod = L.helpers_module(monkeypatch)
    cls = train_loop.device_trainer(mod.Trainer)
    cls.step_class, cls.max_bytes, cls.virtual_ranks = step or L.FakeStep, None, K
    table = L.make_table(str(tmp_path / "data"), 13, "onex")
    exp = L.Exp(table, "onex", str(tmp_path / "out"), world=world, rank=rank, max_epoch=2, build=L.tiny_build)
    exp.evaluator = _recording_evaluator() if evaluator is None else evaluator
    t = cls(exp, L.args_for(batch_size=batch_size))
    t.train()
    return t, exp, mod, (step or L.FakeStep).log


@pytest.mark.parametrize("world,K", [(1, 2), (2, 2), (1, 4)])
def test_device_trainer_feeds_every_virtual_rank_its_stream(tmp_path, monkeypatch, world, K):
    """over two epochs, every replay holds the batches of ranks rank*K .. rank*K + K - 1 of a W x K-rank run side by
    side, each what a fresh YoloBatchSampler over rank g's InfiniteSampler yields; the Trainer runs K virtual ranks"""
    import test_train_loop as L
    G, B = world * K, 1
    for rank in range(world):
        ev = types.SimpleNamespace(evaluate_virtual_ranks=lambda *a, **kw: (0.0, 0.0, "summary"))   # no process group
        t, exp, _, log = _loop(tmp_path / f"r{rank}", monkeypatch, K, world, rank, G * B, evaluator=ev)
        assert t.tr.virtual_ranks == K
        fresh = [iter(L.YoloBatchSampler(sampler=L.InfiniteSampler(13, rank=rank * K + k, world_size=G), batch_size=B,
                                         drop_last=False, mosaic=False)) for k in range(K)]
        assert t.max_iter == len(L.YoloBatchSampler(sampler=L.InfiniteSampler(13, world_size=G), batch_size=B,
                                                    drop_last=False))
        assert len(log.replays) == 2 * t.max_iter
        want = [[int(i) for f in fresh for _, i in next(f)] for _ in range(2 * t.max_iter)]
        assert [L._indices_of(r["slot"], exp.table, 2) for r in log.replays] == want


def test_device_trainer_logs_rank_0_and_evaluates_every_rank_shard(tmp_path, monkeypatch):
    """K = 2, one pair per rank, the real step (kernels emulated): every log line shows virtual rank 0's losses; each
    epoch's evaluation runs virtual rank g's DistributedSampler(num_replicas=2, rank=g) shard in batches of one pair
    with copy g's EMA weights, rank 0 first, and scores the two shards' rows once, concatenated in rank order"""
    K, n_val = 2, 11
    ev = _recording_evaluator(n_val)
    t, exp, mod, log = _loop(tmp_path, monkeypatch, K, 1, 0, K, step=EagerStep, evaluator=ev)
    # the log: rank 0's losses at the print iterations (3, 6 of every epoch), which differ from rank 1's
    lines = [ln for ln in mod.logger.lines if ln.startswith("epoch: ")]
    its = [e * t.max_iter + i for e in range(2) for i in range(exp.print_interval - 1, t.max_iter, exp.print_interval)]
    assert len(lines) == len(its) == 4
    differs = 0
    for ln, i in zip(lines, its):
        r0, r1 = log.rank_rows[i]
        for k in ("total_loss", "iou_loss", "l1_loss", "conf_loss", "cls_loss"):
            assert "{}: {:.1f}".format(k, r0[k]) in ln, (i, k, ln)
            differs += "{}: {:.1f}".format(k, r1[k]) not in ln
    assert differs > 0
    # the evaluation: per epoch one call per virtual rank, in rank order, then one scoring of the concatenated rows
    assert len(ev.calls) == 2 * K and len(ev.got) == 2
    ds = ev.dataloader.dataset
    for k in range(K):
        idx = [int(i) for i in torch.utils.data.distributed.DistributedSampler(ds, num_replicas=K, rank=k, shuffle=False)]
        assert ev.calls[K + k]["batches"] == [[i] for i in idx]
    order = [i for k in range(K) for b in ev.calls[K + k]["batches"] for i in b]
    assert [d["image_id"] for d in ev.got[1][0]] == order
    assert ev.got[1][1][2] == sum(len(ev.calls[K + k]["batches"]) - 1 for k in range(K))
    for k in range(K):                                  # the last epoch's calls held copy k's EMA weights
        want = t.tr.ema_state_dict(k)
        assert all(torch.equal(ev.calls[K + k]["state"][n], v) for n, v in want.items())
    name = next(n for n, v in want.items() if "running_mean" in n)
    assert not torch.equal(ev.calls[K]["state"][name], ev.calls[K + 1]["state"][name])
    assert ev.batches == [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9, 10]]   # the loader's own batches again afterwards


def test_device_trainer_virtual_rank_refusals(tmp_path, monkeypatch):
    """a batch that leaves a virtual rank no sample, a sampler other than yolox's InfiniteSampler, and an evaluator
    that cannot evaluate one shard per virtual rank"""
    import test_train_loop as L
    with pytest.raises(ValueError, match="no sample"):
        _loop(tmp_path / "a", monkeypatch, 4, 1, 0, 3)
    with pytest.raises(ValueError, match="Evaluator"):
        _loop(tmp_path / "c", monkeypatch, 2, 1, 0, 2, evaluator=L.Evaluator())

    class Other(L.InfiniteSampler):
        pass

    monkeypatch.setattr(L, "InfiniteSampler", Other)
    with pytest.raises(ValueError, match="Other"):
        _loop(tmp_path / "b", monkeypatch, 2, 1, 0, 2)
    from streamyolo_b200 import dropin
    with pytest.raises(ValueError, match="virtual_ranks"):
        dropin.install_trainer(0)
