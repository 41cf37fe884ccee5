"""The gradient arithmetic of grad_mode MLP_TC_HALF (csrc/render_bwd.cu, render_bwd_tc_kernel) in plain PyTorch.

`mlp_grad_emulated(x, w)` is an `mlp_fn` for oracle.render_samples / render_rays.  Its forward is exactly oracle.mlp.
In its backward, every nn.Linear rounds the three GEMM operands -- dpre (the gradient at the pre-activation), the
layer input x and the weight W -- to an 11-bit significand (round to nearest even) with an unbounded exponent, which is
what an fp16 operand with an exact per-tile power-of-two scale holds, and accumulates dx = dpre W and dW = dpre^T x in
fp64.  Bias gradients are fp64 sums of the unrounded dpre.  Everything outside the linears (ReLU, the modulation
product, sigmoid, compositing, the volume gather) is ordinary fp32 autograd, as in the kernel."""
import torch
import torch.nn.functional as F


def round_half_significand(t):
    """fp64 copy of `t` rounded to 11 significant bits (fp16's significand), exponent unchanged."""
    m, e = torch.frexp(t.double())
    return torch.ldexp(torch.round(m * 2048.0) / 2048.0, e.double())


class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, rounding):
        ctx.save_for_backward(x, weight)
        ctx.rounding = rounding
        return F.linear(x, weight, bias)

    @staticmethod
    def backward(ctx, g):
        x, weight = ctx.saved_tensors
        r = round_half_significand if ctx.rounding else (lambda t: t.double())
        gd, xd, wd = r(g), r(x), r(weight)
        dx = (gd @ wd).to(x.dtype)
        dw = (gd.reshape(-1, g.shape[-1]).t() @ xd.reshape(-1, x.shape[-1])).to(weight.dtype)
        db = g.double().reshape(-1, g.shape[-1]).sum(0).to(weight.dtype)
        return dx, dw, db, None


def mlp_grad_emulated(x, w, rounding=True):
    """oracle.mlp with the backward of grad_mode MLP_TC_HALF (rounding=False: the same with exact operands)."""
    pe, feat, dirs = x[..., :63], x[..., 63:83], x[..., 83:86]
    p = "mlp/nerf."

    def lin(t, name):
        return _Linear.apply(t, w[p + name + ".weight"], w[p + name + ".bias"], rounding)
    mod = lin(feat, "pts_bias")
    h = pe
    for i in range(6):
        h = F.relu(lin(h, f"pts_linears.{i}") * mod)
        if i == 4:
            h = torch.cat([pe, h], -1)
    sigma = F.relu(lin(h, "alpha_linear"))
    f = lin(h, "feature_linear")
    hv = F.relu(lin(torch.cat([f, dirs], -1), "views_linears.0"))
    rgb = torch.sigmoid(lin(hv, "rgb_linear"))
    return torch.cat([rgb, sigma], -1)
