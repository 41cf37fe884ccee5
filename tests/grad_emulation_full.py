"""The arithmetic of grad_mode GRAD_TC_FULL (csrc/render_bwd.cu, render_bwd_tc_kernel with tile_mlp_tc) in plain
PyTorch.

`mlp_full_emulated(x, w)` is an `mlp_fn` for oracle.render_samples.  Its forward is the tensor-core recompute: every
GEMM of N >= 64 takes fp16 operands -- the encoding and the 20 features unscaled, hidden activations and f with a
power-of-two scale per row that puts the row's max |v| in [2^14, 2^15), weights unscaled -- and accumulates exactly
(fp64), rounded once to fp32 before the bias.  The heads of width <= 3 (alpha_linear, rgb_linear, the view-direction
columns of views_linears.0) take operands rounded to fp16's significand with an unbounded exponent (round_half).
Biases, the modulation product, ReLU and sigmoid are fp32.  Its backward is MLP_TC_HALF's (grad_emulation._Linear):
dpre, x and W rounded to an 11-bit significand, fp64 accumulation, bias gradients from the unrounded dpre."""
import torch
import torch.nn.functional as F

from grad_emulation import _Linear, round_half_significand

FP16_MAX = 65504.0


def row_scaled_half(v):
    """fp64 value of the fp16 operand of `v` [..., K] with a power-of-two scale 2^e per row: max|row| * 2^e in
    [2^14, 2^15), e = 0 for a zero row, e clamped to [-62, 62]; conversions saturate."""
    v = v.float()
    m = v.abs().amax(-1, keepdim=True)
    e = torch.where(m > 0, 14 - (torch.frexp(m).exponent - 1), torch.zeros_like(m, dtype=torch.int32)).clamp(-62, 62)
    s = torch.ldexp(torch.ones_like(m), e)
    return (v * s).clamp(-FP16_MAX, FP16_MAX).half().double() / s.double()


def _operand(t, kind):
    if kind == "front":
        return t.float().clamp(-FP16_MAX, FP16_MAX).half().double()
    if kind == "row":
        return row_scaled_half(t)
    return round_half_significand(t)                                   # "head": FFMA on round_half operands


class _LinearFull(_Linear):
    """Forward: sum over the K-groups `parts` = ((k0, k1, kind), ...) of operand(x[..., k0:k1]) operand(W[:, k0:k1])^T
    in fp64, rounded to fp32, plus the fp32 bias.  Backward: MLP_TC_HALF's."""
    @staticmethod
    def forward(ctx, x, weight, bias, parts):
        ctx.save_for_backward(x, weight)
        ctx.rounding = True
        acc = 0.0
        for k0, k1, kind in parts:
            wk = weight[:, k0:k1]
            wq = round_half_significand(wk) if kind == "head" else wk.float().half().double()
            acc = acc + _operand(x[..., k0:k1], kind) @ wq.t()
        return acc.to(x.dtype) + bias


def mlp_full_emulated(x, w):
    """oracle.mlp in the arithmetic of grad_mode GRAD_TC_FULL (forward and backward)."""
    pe, feat, dirs = x[..., :63], x[..., 63:83], x[..., 83:86]
    p = "mlp/nerf."

    def lin(t, name, parts):
        return _LinearFull.apply(t, w[p + name + ".weight"], w[p + name + ".bias"], parts)
    mod = lin(feat, "pts_bias", ((0, 20, "front"),))
    h = pe
    for i in range(6):
        parts = ((0, 63, "front"),) if i == 0 else ((0, 63, "front"), (63, 191, "row")) if i == 5 else ((0, 128, "row"),)
        h = F.relu(lin(h, f"pts_linears.{i}", parts) * mod)
        if i == 4:
            h = torch.cat([pe, h], -1)
    sigma = F.relu(lin(h, "alpha_linear", ((0, 128, "head"),)))
    f = lin(h, "feature_linear", ((0, 128, "row"),))
    hv = F.relu(lin(torch.cat([f, dirs], -1), "views_linears.0", ((0, 128, "row"), (128, 131, "head"))))
    rgb = torch.sigmoid(lin(hv, "rgb_linear", ((0, 64, "head"),)))
    return torch.cat([rgb, sigma], -1)
