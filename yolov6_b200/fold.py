"""Weight preparation for the deploy-form kernels: BatchNorm folding and RepVGG re-parameterisation.

Reference: fuse_conv_and_bn / fuse_model (yolov6/utils/torch_utils.py:50-94) and
RepVGGBlock / QARepVGGBlock[V2].get_equivalent_kernel_bias / switch_to_deploy (yolov6/layers/common.py:257-477).  The
reference does this by mutating modules in fp32; here it is a pure function from the train-form
state_dict to per-op (weight KRSC, bias) pairs, computed in fp64 so the only rounding left is the
final cast (the reference's own fold drifts its outputs by ~1e-4, SURVEY.md A.2).
"""
import torch

from .arch import dp_bn

BN_EPS = 1e-3  # torch_utils.py:41-43


def _bn_affine(sd, p):
    g, b = sd[p + ".weight"].double(), sd[p + ".bias"].double()
    m, v = sd[p + ".running_mean"].double(), sd[p + ".running_var"].double()
    scale = g / torch.sqrt(v + BN_EPS)
    return scale, b - m * scale


def fold_conv_bn(sd, p):
    """conv (no bias) + BN -> (W' [Cout,Cin,k,k], b' [Cout]) in fp64."""
    w = sd[p + ".conv.weight"].double()
    scale, shift = _bn_affine(sd, p + ".bn")
    return w * scale.view(-1, 1, 1, 1), shift


def fold_op(sd, op):
    """Returns (weight fp64 [Cout,kh,kw,Cin] (KRSC), bias fp64 [Cout]); convT returns 4 KRSC 1x1 weights; a depthwise conv
    (op.kind 'dw') returns [C,k,k,1]."""
    n = op.name
    if op.layout == "dp":       # DPBlock conv with bias, then BN: scale * (conv + b) + shift (common.py:926-929)
        scale, shift = _bn_affine(sd, dp_bn(n))
        w = sd[n + ".weight"].double() * scale.view(-1, 1, 1, 1)
        return w.permute(0, 2, 3, 1).contiguous(), sd[n + ".bias"].double() * scale + shift
    if op.layout == "rep":
        k3, b3 = fold_conv_bn(sd, n + ".rbr_dense")
        k1, b1 = fold_conv_bn(sd, n + ".rbr_1x1")
        k = k3 + torch.nn.functional.pad(k1, [1, 1, 1, 1])
        b = b3 + b1
        if n + ".rbr_identity.weight" in sd:
            scale, shift = _bn_affine(sd, n + ".rbr_identity")
            idx = torch.arange(op.cin)
            k[idx, idx, 1, 1] += scale
            b = b + shift
        return k.permute(0, 2, 3, 1).contiguous(), b
    if op.layout == "qa":
        # QARepVGGBlock[V2].get_equivalent_kernel_bias (common.py:348-360, 427-442): K = fold(W3, BN_d) + pad(W1) + I (+ 1/9 on
        # every tap of the diagonal: AvgPool2d(3, 1, 1) counts the zero padding), bias b_d; then the post-sum bn in eval mode
        k, b = fold_conv_bn(sd, n + ".rbr_dense")
        k = k + torch.nn.functional.pad(sd[n + ".rbr_1x1.weight"].double(), [1, 1, 1, 1])
        if op.identity:
            idx = torch.arange(op.cin)
            k[idx, idx, 1, 1] += 1.0
            if op.avg:
                k[idx, idx] += 1.0 / 9.0
        scale, shift = _bn_affine(sd, n + ".bn")
        k = k * scale.view(-1, 1, 1, 1)
        return k.permute(0, 2, 3, 1).contiguous(), b * scale + shift
    if op.layout == "cba":
        k, b = fold_conv_bn(sd, n + ".block")
        return k.permute(0, 2, 3, 1).contiguous(), b
    if op.layout == "cm":       # rows [w_row0, w_row0 + cout) of a bare ConvModule (arch.Op.w_row0)
        k, b = fold_conv_bn(sd, n)
        r = slice(op.w_row0, op.w_row0 + op.cout)
        return k[r].permute(0, 2, 3, 1).contiguous(), b[r]
    if op.layout == "plain":
        return sd[n + ".weight"].double().permute(0, 2, 3, 1).contiguous(), sd[n + ".bias"].double()
    if op.layout == "convT":
        w = sd[n + ".upsample_transpose.weight"].double()          # [Cin, Cout, 2, 2]
        quads = [w[:, :, dy, dx].t().contiguous().view(op.cout, 1, 1, op.cin) for dy in range(2) for dx in range(2)]
        return quads, sd[n + ".upsample_transpose.bias"].double()
    raise ValueError(op.layout)


def se_weights(sd, op):
    """SEBlock FCs, unfolded (common.py:745-757): (w1 [Cr, C], b1 [Cr], w2 [C, Cr], b2 [C]) in fp64."""
    n = op.name
    return (sd[n + ".conv1.weight"].double().flatten(1), sd[n + ".conv1.bias"].double(),
            sd[n + ".conv2.weight"].double().flatten(1), sd[n + ".conv2.bias"].double())
