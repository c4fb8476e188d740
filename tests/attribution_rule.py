"""Host restatements for the DeepLift / DeepLiftShap / GradientShap statement scores (not a test module).

The draws of ``ddfa_stmt_shap_input`` (include/ddfa_b200.h) from the host Philox4x32-10 of head_batches.py, and the three rules
on the fp64 oracle with torch.autograd: captum's ``DeepLift`` rescale rule at each ``nn.ReLU`` of the MLP head (every other
nonlinearity a plain gradient), the mean over baselines of ``DeepLiftShap``, and ``GradientShap``'s mean over samples of
(x~ - b) * grad at b + alpha (x~ - b).
"""
import numpy as np
import torch
from torch import nn

from head_batches import philox4x32_10
from statement_rule import oracle_input_grad

BASE_WORD, ALPHA_WORD = 0x40000000, 0x80000000
RESCALE_EPS = 1e-10          # captum's DeepLift eps: below it the plain derivative is kept


def _words(seed: int, batch: int, sample: int, index, column):
    index = np.asarray(index, dtype=np.uint64)
    z = np.zeros(index.shape, dtype=np.uint64)
    return philox4x32_10((z + np.uint64(batch & 0xFFFFFFFF), z + np.uint64(sample), index, z + np.asarray(column, dtype=np.uint64)),
                         (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))


def alphas(seed: int, batch: int, sample: int, num_graphs: int) -> np.ndarray:
    """α_b of every function: (w0 >> 8) 2^-24 of the counter (batch, sample, b, ALPHA_WORD); exact in float32."""
    w0 = _words(seed, batch, sample, np.arange(num_graphs), ALPHA_WORD)[0]
    return ((w0 >> np.uint64(8)).astype(np.float64) * 2.0 ** -24).astype(np.float32)


def gaussians(seed: int, batch: int, sample: int, num_nodes: int, dim: int, baseline: bool) -> np.ndarray:
    """ε [N, dim] in float64: Box-Muller on the word pairs of the counters (batch, sample, n, q [| BASE_WORD]), columns 4q..4q+3."""
    q = np.arange(dim // 4, dtype=np.uint64)
    n = np.arange(num_nodes, dtype=np.uint64)
    nn_, qq = np.meshgrid(n, q, indexing="ij")
    w = _words(seed, batch, sample, nn_, qq | np.uint64(BASE_WORD if baseline else 0))
    out = np.empty((num_nodes, dim // 4, 4))
    for k, (a, b) in enumerate(((w[0], w[1]), (w[2], w[3]))):
        u1 = ((a >> np.uint64(8)) + np.uint64(1)).astype(np.float64) * 2.0 ** -24
        u2 = (b >> np.uint64(8)).astype(np.float64) * 2.0 ** -24
        r = np.sqrt(-2.0 * np.log(u1))
        out[:, :, 2 * k] = r * np.cos(2 * np.pi * u2)
        out[:, :, 2 * k + 1] = r * np.sin(2 * np.pi * u2)
    return out.reshape(num_nodes, dim)


def rescale_multiplier(z, z_ref, branch=None):
    """captum's `nonlinear` rule for relu: (relu(z) - relu(z')) / (z - z'), or the derivative [z > 0] (``branch`` when given:
    the side a forward took) where |z - z'| < RESCALE_EPS."""
    dz = z - z_ref
    plain = (z > 0).to(z.dtype) if branch is None else branch.to(z.dtype)
    small = dz.abs() < RESCALE_EPS
    return torch.where(small, plain, (torch.relu(z) - torch.relu(z_ref)) / torch.where(small, torch.ones_like(dz), dz))


class _RescaledReLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z, z_ref):
        ctx.save_for_backward(z, z_ref)
        return torch.relu(z)

    @staticmethod
    def backward(ctx, g):
        z, z_ref = ctx.saved_tensors
        return g * rescale_multiplier(z, z_ref), None


def head_rescaled(o, pooled, pooled_ref):
    """The oracle's MLP head on ``pooled`` with each hidden ReLU's gradient under the rescale rule against ``pooled_ref``."""
    layers = [m for m in o.output_layer if isinstance(m, nn.Linear)]
    h, hr = pooled, pooled_ref.detach()
    for i, lin in enumerate(layers):
        z = lin(h)
        if i == len(layers) - 1:
            return z.reshape(-1)
        with torch.no_grad():
            zr = lin(hr)
        h, hr = _RescaledReLU.apply(z, zr), torch.relu(zr)


def _pooled(o, g, x):
    return o.pooling(g, torch.cat([o.ggnn(g, x), x], -1))


def oracle_deeplift(o, g, baselines):
    """DeepLiftShap over ``baselines`` (a list of [N, D] tensors; one zero tensor: DeepLift): the mean over j of
    Σ_d (x - b_j) · g~_j, g~_j the input gradient with the head's ReLUs rescaled against the forward from b_j."""
    with torch.no_grad():
        x = o.embed(g)
    acc = torch.zeros_like(x)
    for b in baselines:
        with torch.no_grad():
            ref = _pooled(o, g, b)
        xg = x.detach().clone().requires_grad_(True)
        head_rescaled(o, _pooled(o, g, xg), ref).sum().backward()
        acc += (x - b) * xg.grad
    return (acc / len(baselines)).sum(1)


def oracle_gradient_shap(o, g, seed: int, batch: int, samples: int, noise_stdev: float = 0.0, baseline_stdev: float = 0.0):
    """GradientShap with the device's draws: per sample s, x~ = x + noise ε, b = baseline ε', α_b per function; the mean over s of
    Σ_d (x~ - b) · ∂logit/∂x at b + α (x~ - b)."""
    with torch.no_grad():
        x = o.embed(g)
    N, D = x.shape
    bnn = g.batch_num_nodes()
    gid = torch.repeat_interleave(torch.arange(bnn.numel()), bnn)
    acc = torch.zeros_like(x)
    for s in range(samples):
        xt = x + noise_stdev * torch.from_numpy(gaussians(seed, batch, s, N, D, False)) if noise_stdev > 0 else x
        b = baseline_stdev * torch.from_numpy(gaussians(seed, batch, s, N, D, True)) if baseline_stdev > 0 else torch.zeros_like(x)
        a = torch.from_numpy(alphas(seed, batch, s, bnn.numel()).astype(np.float64))[gid][:, None]
        acc += (xt - b) * oracle_input_grad(o, g, b + a * (xt - b))
    return (acc / samples).sum(1)
