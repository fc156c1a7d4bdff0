"""CPU ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

``ActOracle``: ``streamyolo_oracle.StreamYoloOracle`` with every yolox BaseConv's activation chosen by name, as
``act=`` of the reference's constructors selects it through [yolox] ``get_activation``: "silu" (``nn.SiLU``), "relu"
(``nn.ReLU``) or "lrelu" (``nn.LeakyReLU(0.1)``).  Same storage-precision hook ``q``, applied at the same places.
Pinned against outputs of the unmodified reference by ``oracle/make_act_golden.py`` / ``tests/test_activations.py``.
"""
import torch
import torch.nn.functional as F

from oracle.streamyolo_oracle import StreamYoloOracle

ACTIVATIONS = {"silu": F.silu, "relu": F.relu, "lrelu": lambda t: F.leaky_relu(t, 0.1)}


class ActOracle(StreamYoloOracle):
    def __init__(self, cfg, state, q=None, act="silu"):
        super().__init__(cfg, state, q)
        self.act = ACTIVATIONS[act]

    def base_conv(self, pfx, x, k, stride, res=None, round_out=True):
        """yolox BaseConv = act(BN(Conv2d(bias=False, pad=(k-1)//2))) [+ residual] (StreamYoloOracle.base_conv with the
        activation of this oracle)."""
        P, q, c = self.P, self.q, self.cfg
        self._note(pfx + ".in", x)
        if res is not None:
            self._note(pfx + ".res", res)
        y = F.conv2d(x, q(P[pfx + ".conv.weight"]), None, stride, (k - 1) // 2)
        g, b = P[pfx + ".bn.weight"], P[pfx + ".bn.bias"]
        if self.training:
            y = q(y)
            n = y.numel() // y.shape[1]
            mean = y.mean((0, 2, 3))
            var = y.var((0, 2, 3), unbiased=False)
            m = c.bn_momentum
            P[pfx + ".bn.running_mean"].mul_(1 - m).add_(m * mean)
            P[pfx + ".bn.running_var"].mul_(1 - m).add_(m * var * (n / max(n - 1, 1)))
            P[pfx + ".bn.num_batches_tracked"] += 1
        else:
            mean, var = P[pfx + ".bn.running_mean"], P[pfx + ".bn.running_var"]
        scale = g * torch.rsqrt(var + c.bn_eps)
        shift = b - mean * scale
        y = self.act(y * scale[None, :, None, None] + shift[None, :, None, None])
        self._note(pfx, y)
        if res is not None:
            y = y + res
        if round_out:
            y = q(y)
        self._note(pfx + ".out", y)
        return y
