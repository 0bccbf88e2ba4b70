"""fp64 oracle of the mish and gelu MLP nonlinearities -- TEST INFRASTRUCTURE.

oracle/nn_ref.ScalarMLPFunction restates nequip's ScalarMLPFunction with SiLU between layers (SURVEY appendix A.3).  This
module restates the same class for every nonlinearity the reference builder documents (allegro_models.py: silu, mish,
gelu or None) and installs it into oracle.nn_ref while an oracle model is built, so AllegroOracle takes
``scalar_embed_mlp_nonlinearity`` / ``allegro_mlp_nonlinearity`` / ``readout_mlp_nonlinearity`` = "mish" / "gelu".

nequip's own definitions are parity unpinned, as SiLU's gain already is (DESIGN section 2):
  * the gain of the layer after an activation is the second-moment gain 1/sqrt(E_{z~N(0,1)}[phi(z)^2]), by the trapezoid
    rule on [-12, 12] with 240 001 points, as ``silu_second_moment_gain``: silu 1.676532, mish 1.486848, gelu 1.533530;
  * gelu is the exact erf form, x Phi(x) (``torch.nn.functional.gelu`` default).  The tanh approximation has gain
    1.533581; the gain cannot tell the two apart, so the form is a stated choice.
For SiLU the class is the oracle's own, bit for bit: weights are drawn by the parent in the same order, and the gains and
the activation of a SiLU MLP are the parent's.
"""
import contextlib
import math

import numpy as np
import torch

from oracle import model_ref
from oracle import nn_ref as R


def _gain(phi) -> float:
    z = np.linspace(-12.0, 12.0, 240001)
    w = np.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)
    s = phi(z)
    return float(1.0 / math.sqrt(np.trapezoid(s * s * w, z)))


def _mish_np(z):
    return z * np.tanh(np.logaddexp(0.0, z))


def _gelu_np(z):
    from scipy.special import erfc

    return 0.5 * z * erfc(-z / math.sqrt(2))


GAINS = {"silu": R._SILU_GAIN, "mish": _gain(_mish_np), "gelu": _gain(_gelu_np)}
PHI = {"silu": torch.nn.functional.silu, "mish": torch.nn.functional.mish, "gelu": torch.nn.functional.gelu}


def dphi(name, x):
    """phi'(x) in closed form (the table of the C ABI header)."""
    if name == "silu":
        s = torch.sigmoid(x)
        return s * (1 + x * (1 - s))
    if name == "mish":
        t = torch.tanh(torch.nn.functional.softplus(x))
        return t + x * (1 - t * t) * torch.sigmoid(x)
    return 0.5 * torch.erfc(-x / math.sqrt(2)) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def dphi_scale(name, x):
    """The sum of the absolute values of the two terms phi'(x) is formed from (the closed forms above): the scale of the
    rounding error of any evaluation of phi'(x), which is not small relative to phi'(x) itself near its zero."""
    if name == "silu":
        s = torch.sigmoid(x)
        return s + (x * s * (1 - s)).abs()
    if name == "mish":
        t = torch.tanh(torch.nn.functional.softplus(x))
        return t.abs() + (x * (1 - t * t) * torch.sigmoid(x)).abs()
    return 0.5 * torch.erfc(-x / math.sqrt(2)) + (x * torch.exp(-0.5 * x * x)).abs() / math.sqrt(2 * math.pi)


class ScalarMLPFunction(R.ScalarMLPFunction):
    """R.ScalarMLPFunction with nonlinearity in {silu, mish, gelu, None}."""

    def __init__(self, input_dim, output_dim, hidden_layers_depth=0, hidden_layers_width=None, nonlinearity="silu", bias=False,
                 forward_weight_init=True):
        assert nonlinearity is None or nonlinearity in PHI
        super().__init__(input_dim, output_dim, hidden_layers_depth, hidden_layers_width, None if nonlinearity is None else "silu", bias,
                         forward_weight_init)
        self.nonlinearity = nonlinearity
        gain = 1.0
        self.alphas = []
        for h_in, h_out in zip(self.dims, self.dims[1:]):
            self.alphas.append(gain / math.sqrt(h_in if forward_weight_init else h_out))
            gain = GAINS[nonlinearity] if nonlinearity is not None else 1.0

    def forward(self, x):
        n = len(self.weights)
        for k, (w, a) in enumerate(zip(self.weights, self.alphas)):
            x = x @ (a * w)
            if k < n - 1 and self.nonlinearity is not None:
                x = PHI[self.nonlinearity](x)
        return x


@contextlib.contextmanager
def nonlinearities():
    """oracle.nn_ref builds its MLPs with the class above inside this block."""
    prev = R.ScalarMLPFunction
    R.ScalarMLPFunction = ScalarMLPFunction
    try:
        yield
    finally:
        R.ScalarMLPFunction = prev


def oracle(**kw):
    """AllegroOracle(**kw) with any of the three nonlinearity kwargs."""
    with nonlinearities():
        return model_ref.AllegroOracle(**kw)
