"""GPU: graph replays of the training step with the host running ahead of the device.

A graphed training loop need not wait for the device between steps: ``Trainer.replay`` / ``replay_size`` return device
tensors, the next batch is copied into the static inputs on the device, and the next replay is enqueued at once.  Each
replay's learning rate and EMA decay reach the captured optimiser step through a device block that the host refills
before every replay, so a step still queued behind others must run with its own values.  These tests replay with no host
synchronisation between the steps, a different learning rate and batch per step, and compare with eager
``Trainer.step`` bit for bit."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.make_golden import CASES  # noqa: E402
from streamyolo_b200 import synth, train  # noqa: E402
from test_gpu_model import build_product  # noqa: E402

C = CASES["tiny_120x160"]
STEPS = 10
LRS = [1e-4 * (1 + 0.1 * i) for i in range(STEPS)]


def _batches(sizes):
    """one batch per step, all on the device before the loop (a copy from pageable host memory synchronises the host)"""
    out = []
    for i, (h, w) in enumerate(sizes):
        x = synth.synth_frames(C["B"], h, w, seed=100 + i).cuda()
        out.append((x, tuple(t.cuda() for t in synth.synth_labels(C["B"], h, w, seed=200 + i))))
    torch.cuda.synchronize()
    return out


def _clone(batch):
    return batch[0].clone(), tuple(t.clone() for t in batch[1])


def _load(static, batch):
    static[0].copy_(batch[0])
    for dst, src in zip(static[1], batch[1]):
        dst.copy_(src)


def _trainer():
    return train.Trainer(build_product(C["depth"], C["width"]).train(), lr=LRS[0])


def _eager(batches):
    tr = _trainer()
    losses = [tr.step(x, tg, lr=lr)["total_loss"].clone() for (x, tg), lr in zip(batches, LRS)]
    torch.cuda.synchronize()
    return tr, losses


def _assert_same(ta, tb, want, got):
    torch.cuda.synchronize()
    assert torch.equal(torch.stack(got), torch.stack(want)), (got, want)
    assert tb.updates == ta.updates == STEPS
    assert torch.equal(tb.fs.state, ta.fs.state), "fs.state"
    assert torch.equal(tb.fs.mom, ta.fs.mom), "fs.mom"
    assert torch.equal(tb.fs.ema, ta.fs.ema), "fs.ema"


def test_replay_without_host_sync_equals_eager_steps():
    batches = _batches([(C["H"], C["W"])] * STEPS)
    ta, want = _eager(batches)
    tb = _trainer()
    static = _clone(batches[0])
    tb.capture(*static)                                  # runs step 1 eagerly (warm-up) at lr = LRS[0], then captures
    got = []
    for batch, lr in zip(batches[1:], LRS[1:]):
        _load(static, batch)
        got.append(tb.replay(lr=lr)["total_loss"].clone())
    _assert_same(ta, tb, want[1:], got)


def test_replay_size_without_host_sync_equals_eager_steps():
    sizes = [(96, 160), (128, 224)]
    seq = [sizes[i % 2] for i in range(STEPS)]
    batches = _batches(seq)
    ta, want = _eager(batches)
    tb = _trainer()
    static = {s: _clone(batches[i]) for i, s in enumerate(sizes)}
    tb.capture_sizes(sizes, static.__getitem__)          # leaves the state as it was: every step is a replay
    got = []
    for s, batch, lr in zip(seq, batches, LRS):
        _load(static[s], batch)
        got.append(tb.replay_size(s, lr=lr)["total_loss"].clone())
    _assert_same(ta, tb, want, got)
