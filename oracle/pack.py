"""Host packing of an inference engine's weights: the float64 fold of yolov6_b200.fold followed by the engine's operand casts
and layout moves, on the CPU.  This is how InferEngine packed its weights before the fold ran on the device
(yolov6_b200/refold.py, yv6_fold); the fold's tests hold the device fold and its host replay to it, byte for byte."""
import torch

from yolov6_b200 import ops
from yolov6_b200.engine import pair_view_candidate, siblings, stem_channels, window_weights
from yolov6_b200.fold import fold_op, se_weights, to_f16


def pack(g, sd, precision):
    """{op index: {key: CPU tensor (a list of them for "w"), "alpha": float}}: InferEngine.weights of graph g at the
    state_dict sd in `precision` ("bf16", "fp16" or "fp32"); raises fold.to_f16's ValueError in fp16 for an out-of-range
    weight."""
    sd = {k: v.detach().cpu() for k, v in sd.items()}
    f16, nsplit = precision == "fp16", 3 if precision == "fp32" else 1

    def planes(w, name):  # KRSC weights in the precision's operand layout (folded in fp64, rounded once)
        if f16:
            return to_f16(w, name).contiguous()
        w = w.float()
        return ops.split3(w).contiguous() if nsplit == 3 else w.to(torch.bfloat16).contiguous()

    weights = {}
    sibling = siblings(g)
    for i, op in enumerate(g.ops):
        if op.kind in ("pool", "shuffle", "up") or (op.kind == "pred" and op.head[0] not in ("cls", "reg")):
            continue
        if op.kind == "se":
            weights[i] = dict(zip(("w1", "b1", "w2", "b2"), (t.float().contiguous() for t in se_weights(sd, op))))
            continue
        w, b = fold_op(sd, op)
        ent = {}
        if op.kind == "stem":
            cp = stem_channels(g, op)
            w, b = torch.cat([w, w.new_zeros((cp - op.cout,) + w.shape[1:])]), torch.cat([b, b.new_zeros(cp - op.cout)])
            if f16:
                to_f16(w, op.name)
            ent["w_dev"] = w.float().permute(1, 2, 3, 0).contiguous()
            ent["b_dev"] = b.float().contiguous()
        elif op.kind == "dw":
            ent["w_dev"] = w[..., 0].permute(1, 2, 0).reshape(op.k * op.k, op.cin).float().contiguous()
            ent["b_dev"] = b.float().contiguous()
        else:
            w = w if op.kind == "convT" else window_weights(g, op, w)
            ws = w if isinstance(w, list) else [w]
            ent["w"] = [planes(wi, op.name) for wi in ws]
            if pair_view_candidate(op):
                ent["w_pair"] = planes(ops.pair_view_weights(ws[0]), op.name)
            ent["bias"] = ops.pad_bias(b, op.cout)
        ent["alpha"] = float(sd[op.alpha]) if (op.alpha and op.res is not None) else 1.0
        weights[i] = ent
    for i, j in sibling.items():
        (wa, ba), (wb, bb) = fold_op(sd, g.ops[i]), fold_op(sd, g.ops[j])
        weights[i]["w_fused"] = planes(torch.cat([wa, wb], 0), g.ops[i].name)
        weights[i]["bias_fused"] = ops.pad_bias(torch.cat([ba, bb]), 2 * g.ops[i].cout)
    return weights


def tensors(weights):
    """[(op index, key, tensor)] of a packing (InferEngine.weights or pack()), in a fixed order, alpha aside."""
    out = []
    for i in sorted(weights):
        for key in sorted(weights[i]):
            v = weights[i][key]
            if key == "alpha":
                continue
            for q, t in enumerate(v if isinstance(v, list) else [v]):
                out.append((i, f"{key}[{q}]" if isinstance(v, list) else key, t))
    return out
