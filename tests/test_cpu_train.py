"""CPU: the H100-native training step (streamyolo_b200/train.py: flat fp32 state, gradient sink writing into the flat
buffer in walk order, bucketed all-reduce launched from the walk, fused optimiser step) with every kernel replaced by its
torch emulation (tests/emul_ops.py), against the same step made of stock PyTorch pieces (torch.optim.SGD with the
reference's three parameter groups, the Python ModelEMA, a post-hoc all-reduce) -- the semantics of the reference's trainer
loop, /root/reference/exps/train_utils/double_trainer.py:99-123, 171-175."""
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_ops  # noqa: E402
import test_cpu_backward as T  # noqa: E402
from oracle.make_golden import CASES  # noqa: E402
from streamyolo_b200 import ops, synth, train  # noqa: E402
from streamyolo_b200.model import backward, engine  # noqa: E402


def test_flat_state_keeps_the_module_surface(monkeypatch):
    """Re-pointing parameters / buffers into the flat buffers must not change what the reference's tooling sees:
    state_dict keys / values, parameter count, optimizer grouping; gradients are views of the flat gradient buffer and the
    conv1 | conv2 pair of every CSPLayer is adjacent (one weight-gradient launch covers both)."""
    emul_ops.install(monkeypatch, exact=True)
    c = CASES["tiny_120x160"]
    model = T.build_product(c)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    fs = train.FlatState(model)
    after = model.state_dict()
    assert list(after) == list(before)
    for k in before:
        assert torch.equal(after[k], before[k]), k
    n = sum(p.numel() for p in model.parameters())
    assert fs.n_param >= n and fs.n_param - n < 64 * (3 * len(list(model.parameters())))
    base = fs.state.data_ptr()
    for p in model.parameters():
        o, m = fs.offset[id(p)]
        assert p.data_ptr() == base + 4 * o and p.grad.data_ptr() == fs.grad.data_ptr() + 4 * o and m == p.numel()
        assert (o >= fs.decay_begin) == (p.dim() == 4)          # conv weights (incl. the prediction convs) decay, the rest not
    csp = model.backbone.C3_p4
    o1, n1 = fs.offset[id(csp.conv1.conv.weight)]
    assert fs.offset[id(csp.conv2.conv.weight)][0] == o1 + n1
    # walk order: head level 2 first, the stem last
    first = fs.offset[id(model.head.cls_convs[2][1].conv.weight)][0]
    last = fs.offset[id(model.backbone.backbone.stem.conv.conv.weight)][0]
    assert fs.decay_begin <= first < last
    ids = [id(p) for g in train.build_optimizer(model, 0.01).param_groups for p in g["params"]]
    assert sorted(ids) == sorted(id(p) for p in model.parameters())


@pytest.mark.parametrize("name", ["tiny_120x160", "l_depth_64x96"])
def test_launch_plan_matches_recording_forward(name, monkeypatch):
    """train.conv_groups_forward_order -- the list FlatState's layout, the gradient buckets and the batched re-pack are built
    from -- is the conv launch groups of the recording forward in order of first launch; every group runs once except the
    DFP jian convs (jian(cur) and jian(sup): two launches)."""
    emul_ops.install(monkeypatch, exact=True)
    c = CASES[name] if name in CASES else T.DEPTH_CASES[name]
    model = T.build_product(c)
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tape, _ = backward._record(model, x, synth.synth_labels(c["B"], c["H"], c["W"]))
    seen, recorded = set(), []
    for r in tape.ops:
        if r["t"] == "conv" and id(r["mods"][0]) not in seen:
            seen.add(id(r["mods"][0]))
            recorded.append(tuple(map(id, r["mods"])))
    plan = train.conv_groups_forward_order(model)
    assert recorded == [tuple(map(id, g)) for g in plan]
    net = model.backbone
    jian = {id(net.jian2), id(net.jian1), id(net.jian0)}
    assert {id(g[0]): tape.uses[id(g[0])] for g in plan} == {id(g[0]): 2 if id(g[0]) in jian else 1 for g in plan}


def test_trainer_step_matches_stock_pytorch_step(monkeypatch):
    """Three steps of train.Trainer (flat state + fused kernel emulation) == three steps of train.train_step (torch SGD
    nesterov with weight-decay groups + Python ModelEMA): losses, every parameter, the EMA copy and the BatchNorm buffers."""
    emul_ops.install(monkeypatch, exact=True)
    c = CASES["tiny_120x160"]
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"])
    ref = T.build_product(c)
    opt = train.build_optimizer(ref, lr=2e-4)
    ema = train.ModelEMA(ref)
    model = T.build_product(c)
    tr = train.Trainer(model, lr=2e-4)
    assert len(tr.fs.params) == len(list(ref.parameters()))
    wants = [train.train_step(ref, opt, x, tg, ema) for _ in range(3)]     # (not interleaved: the operand caches share one epoch)
    for i in range(3):
        want = wants[i]
        got = tr.step(x, tg)
        d3 = model.backbone.backbone.dark3[0]
        assert any(g[0] is d3 and d3._pk is fwd for g, fwd, _ in tr._packed_groups)      # the batched re-pack feeds the forward
        # ... under the key the forward looks it up with (a lookup with any other key would re-pack)
        assert engine.packed_operand(d3, "_pk", [d3.conv.weight], ops.pack_conv_weight) is d3._pk
        assert abs(float(got["total_loss"]) - float(want["total_loss"])) <= 1e-5 * abs(float(want["total_loss"])), i
    assert tr.sink.launched and sum(b - a for a, b in tr.sink.launched) == tr.fs.n_param      # every gradient in one bucket
    for (k, p), q in zip(model.named_parameters(), ref.parameters()):
        assert torch.allclose(p, q, rtol=1e-5, atol=1e-7), k
    esd, rsd = tr.ema_state_dict(), ema.ema.state_dict()
    assert list(esd) == list(rsd)
    for k in rsd:
        if rsd[k].dtype.is_floating_point:
            assert torch.allclose(esd[k], rsd[k], rtol=1e-5, atol=1e-7), k
    sd, rs = model.state_dict(), ref.state_dict()
    for k in ("backbone.backbone.stem.conv.bn.running_mean", "head.stems.0.bn.running_var", "backbone.jian1.bn.num_batches_tracked"):
        assert torch.allclose(sd[k].float(), rs[k].float(), rtol=1e-5, atol=1e-7), k


def test_loss_scale_and_found_inf(monkeypatch):
    """GradScaler semantics folded into the fused step: a loss scale is undone by inv_scale, found_inf skips the update."""
    emul_ops.install(monkeypatch, exact=True)
    c = CASES["tiny_120x160"]
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"])
    a, b = T.build_product(c), T.build_product(c)
    ta, tb = train.Trainer(a, lr=1e-3, use_ema=False), train.Trainer(b, lr=1e-3, use_ema=False)
    ta.step(x, tg)
    tb.step(x, tg, loss_scale=1024.0)
    for (k, p), q in zip(a.named_parameters(), b.parameters()):
        assert torch.allclose(p, q, rtol=1e-4, atol=1e-7), k
    before = tb.fs.state.clone()
    tb.forward_backward(x, tg)
    tb.optimizer_step(found_inf=torch.ones(1))
    assert torch.equal(before[:tb.fs.n_param], tb.fs.state[:tb.fs.n_param])


DDP_WORKER = r"""
import os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
import torch
import emul_ops, test_cpu_backward as T
from oracle.make_golden import CASES
from streamyolo_b200 import dist as d, synth, train


class MP:
    def setattr(self, o, n, v): setattr(o, n, v)
    def setitem(self, dct, k, v): dct[k] = v


rank, local, world = d.init("gloo")
emul_ops.install(MP(), exact=True)
c = CASES["tiny_120x160"]
x = synth.synth_frames(4, c["H"], c["W"])
fut, cur = synth.synth_labels(4, c["H"], c["W"])
lo, hi = d.shard_pairs(4, world, rank)
model = T.build_product(c)
tr = train.Trainer(model, lr=1e-3, bucket_bytes=64 << 10)
tr.forward_backward(x[lo:hi], (fut[lo:hi], cur[lo:hi]))
assert len(tr.sink.launched) > 2, tr.sink.launched            # several buckets, launched from inside the walk
g_sum = tr.fs.grad.clone()                                     # SUM over the ranks (the mean is folded into the fused step)
exp = []
for a, b in ((0, 2), (2, 4)):
    m = T.build_product(c)
    t2 = train.Trainer(m, lr=1e-3, overlap=False)
    t2.world = 1
    t2.forward_backward(x[a:b], (fut[a:b], cur[a:b]))
    if a == 0:
        # same layout in every Trainer of this architecture
        assert t2.fs.n_param == tr.fs.n_param
    exp.append(t2.fs.grad.clone())
want = exp[0] + exp[1]
assert torch.allclose(g_sum, want, rtol=1e-5, atol=1e-7 * float(want.abs().max())), float((g_sum - want).abs().max())
tr.optimizer_step()                                            # mean = 1 / world inside the kernel
m = T.build_product(c)
t3 = train.Trainer(m, lr=1e-3, overlap=False)
t3.world = 1
t3.fs.grad.copy_(0.5 * want)
t3.optimizer_step()
n = tr.fs.n_param                                              # (the BatchNorm buffers behind it moved with tr's forward)
assert torch.allclose(tr.fs.state[:n], t3.fs.state[:n], rtol=1e-5, atol=1e-7)
print("ok", rank)
"""


def test_trainer_bucketed_allreduce_gloo_world2(tmp_path):
    """Row a19 / SURVEY 8e, host side: two gloo ranks, each runs the recording forward + walk on its shard with the FlatSink
    launching one all-reduce per ~64 KB bucket as the walk completes it; the flat gradient buffer must hold the SUM of the
    two shards' gradients, and the fused step (inv_scale = 1 / world) the update of the mean gradient."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "ddp_tr.py"
    script.write_text(DDP_WORKER)
    port = 29700 + os.getpid() % 90
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port),
                   OMP_NUM_THREADS="4")
        procs.append(subprocess.Popen([sys.executable, str(script), root], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=600)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), "\n".join(o[-3000:] for o in outs)
