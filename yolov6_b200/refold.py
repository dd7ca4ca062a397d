"""Folding a train-form state into the weight tensors of a built InferEngine, in place (yv6_fold, include/yv6.h).

The state is read from ONE flat fp32 buffer with a `slots` table {name: (offset, numel, shape)}: a Model's FlatState
(`pflat`), a FusedSGDEMA's `ema`, or a state_dict staged into that form (`stage`).  The work is described by records built
on the host once per (engine, layout) and kept on the device:

  * a channel record per op (yv6_fold_chan): the BatchNorm affine of each branch and the folded bias, in float64;
  * element records (yv6_fold_rec), one per destination region: the conv / pred weights `w` (the Lite 16-aligned channel
    window: engine.window_weights), the column-pair view weights `w_pair` (ops.pair_view_weights, one record per source tap
    column), the fused cls / reg siblings `w_fused` / `bias_fused` (one record per half), the ConvTranspose quadrants, the
    padded biases, the stem's [3][3][3][Cout] fp32 weights (channel padding left zero), the depthwise [k*k][C] weights and
    the SE FCs.

Zero regions of the destinations (bias padding, window columns, the pair view's zero taps, the stem's pad channels) are
never written: the engine allocates them zeroed.  The values are bit for bit those of fold.fold_op's float64 fold followed by
the engine's casts (bf16: .float() then round to nearest even; fp16: through fp32, as torch casts float64; fp32 mode: split3
of the fp32 value; biases: float64 -> fp32).  `replay_host` executes the same records with torch's float64 CPU ops: it is how
an engine on the CPU device (planner tests) is packed, and what the fold's CPU test checks against the host packing.

BottleRep's residual scale `alpha` is a host float baked into the conv descriptors (and so into captured graphs); a refold
from a state whose alpha differs raises AlphaChanged before anything is written.
"""
import ctypes as C
from dataclasses import dataclass, field

import torch

from . import _lib, ops
from ._lib import (FOLD_AVG, FOLD_BF16, FOLD_BIAS, FOLD_C_BIAS, FOLD_C_BN, FOLD_C_DP, FOLD_C_QA, FOLD_C_REP, FOLD_CHUNK, FOLD_COPY,
                   FOLD_F16, FOLD_F32, FOLD_IDENTITY, FOLD_SPLIT3, FOLD_W, FOLD_W_CONVT, FOLD_W_COPY, FOLD_W_QA, FOLD_W_REP, FoldChan,
                   FoldRec)
from .arch import dp_bn
from .fold import BN_EPS, f16_range_error

BN_KEYS = ("weight", "bias", "running_mean", "running_var")


class AlphaChanged(ValueError):
    """A refold source's BottleRep alpha differs from the one baked into the engine's conv descriptors (and captured graphs):
    the engine must be rebuilt (and its pipelines recaptured) instead."""


def packed_ops(g):
    """Indices of the ops with inference weights (the fuse_ab / distillation preds are training only)."""
    return [i for i, op in enumerate(g.ops) if op.kind not in ("pool", "shuffle", "up") and
            not (op.kind == "pred" and op.head[0] not in ("cls", "reg"))]


def allocate(g, precision, device):
    """{op index: {key: zeroed tensor}} in the engine's operand layouts (engine.InferEngine.weights, without alpha)."""
    from .engine import conv_window, pair_view_candidate, siblings, stem_channels
    nsplit = 3 if precision == "fp32" else 1
    wdt = torch.float16 if precision == "fp16" else torch.bfloat16

    def planes(shape):
        return torch.zeros(((3,) if nsplit == 3 else ()) + tuple(shape), dtype=wdt, device=device)

    def f32(*shape):
        return torch.zeros(shape, dtype=torch.float32, device=device)

    out = {}
    for i in packed_ops(g):
        op = g.ops[i]
        if op.kind == "se":
            cr = op.cin // 4
            out[i] = dict(w1=f32(cr, op.cin), b1=f32(cr), w2=f32(op.cin, cr), b2=f32(op.cin))
        elif op.kind == "stem":
            cp = stem_channels(g, op)
            out[i] = dict(w_dev=f32(3, 3, op.cin, cp), b_dev=f32(cp))
        elif op.kind == "dw":
            out[i] = dict(w_dev=f32(op.k * op.k, op.cin), b_dev=f32(op.cin))
        elif op.kind == "convT":
            out[i] = dict(w=[planes((op.cout, 1, 1, op.cin)) for _ in range(4)], bias=ops.bias_buffer(op.cout, device))
        else:
            lo, hi = conv_window(g, op)
            ent = dict(w=[planes((op.cout, op.k, op.k, hi - lo))])
            if pair_view_candidate(op):
                ent["w_pair"] = planes((op.cout, 3, 2, 2 * (hi - lo)))
            ent["bias"] = ops.bias_buffer(op.cout, device)
            out[i] = ent
    for i in siblings(g):
        op = g.ops[i]
        out[i]["w_fused"] = planes((2 * op.cout, op.k, op.k, op.cin))
        out[i]["bias_fused"] = ops.bias_buffer(2 * op.cout, device)
    return out


def stage(sd, device):
    """(flat fp32 buffer on `device`, slots) of the floating-point entries of a state_dict (values are read as fp32, the
    dtype of a Model's state)."""
    keys = [k for k, v in sd.items() if v.is_floating_point()]
    slots, off = {}, 0
    for k in keys:
        v = sd[k]
        slots[k] = (off, v.numel(), tuple(v.shape))
        off += v.numel()
    parts = [sd[k].detach().reshape(-1) for k in keys]
    if len({t.device for t in parts}) == 1:
        flat = torch.cat([t.float() for t in parts]) if parts else torch.zeros(0)
        return flat.to(device), slots
    return torch.cat([t.to(device, torch.float32) for t in parts]), slots


def weight_source(src, device):
    """(flat, slots, integer entries) of a load_weights_ source: a state_dict, a FusedSGDEMA (its EMA and the training model's
    layout; the integer buffers of the live model, as ema_state_dict) or (flat tensor, slots)."""
    if isinstance(src, tuple):
        flat, slots = src
        return flat.to(device), slots, {}
    if hasattr(src, "ema_state_dict"):
        fl = src.flat
        flat = src.ema if src.ema is not None else fl.pflat
        ints = {k: v for k, v in src.model.state_dict().items() if not v.is_floating_point()}
        return flat.to(device), fl.slots, ints
    flat, slots = stage(src, device)
    return flat, slots, {k: v for k, v in src.items() if not v.is_floating_point()}


@dataclass
class FoldPlan:
    """Records of one (graph, precision, layout): `chans` / `recs` as dicts (recs name their destination by engine weight
    key `dst` = (key, op index[, quadrant]) and element offset `off`), `checks` the op name of each fp16 check slot, `n_coef`
    float64 coefficients.  `dev` caches the device tables per engine."""
    chans: list
    recs: list
    checks: list
    n_coef: int
    dev: dict = field(default_factory=dict)


def fold_names(g):
    """Every state entry the fold reads (alpha aside), in a fixed order: the layout signature of a slots table."""
    out = []
    for i in packed_ops(g):
        op = g.ops[i]
        n = op.name
        if op.kind == "se":
            out += [n + s for s in (".conv1.weight", ".conv1.bias", ".conv2.weight", ".conv2.bias")]
        elif op.layout == "dp":
            out += [n + ".weight", n + ".bias"] + [dp_bn(n) + "." + k for k in BN_KEYS]
        elif op.layout == "rep":
            for br in ("rbr_dense", "rbr_1x1"):
                out += [f"{n}.{br}.conv.weight"] + [f"{n}.{br}.bn.{k}" for k in BN_KEYS]
            out += [f"{n}.rbr_identity.{k}" for k in BN_KEYS]
        elif op.layout == "qa":
            out += [n + ".rbr_dense.conv.weight"] + [f"{n}.rbr_dense.bn.{k}" for k in BN_KEYS] + [n + ".rbr_1x1.weight"]
            out += [f"{n}.bn.{k}" for k in BN_KEYS]
        elif op.layout == "cba":
            out += [n + ".block.conv.weight"] + [f"{n}.block.bn.{k}" for k in BN_KEYS]
        elif op.layout == "cm":
            out += [n + ".conv.weight"] + [f"{n}.bn.{k}" for k in BN_KEYS]
        elif op.layout == "plain":
            out += [n + ".weight", n + ".bias"]
        elif op.layout == "convT":
            out += [n + ".upsample_transpose.weight", n + ".upsample_transpose.bias"]
    return out


def layout_key(g, slots):
    """Hashable signature of where the fold's entries lie in a slots table (absent entries: None)."""
    return tuple(slots[n][0] if n in slots else None for n in fold_names(g))


def build_plan(g, precision, slots):
    """FoldPlan of graph g in `precision` over a state laid out as `slots`."""
    from .engine import conv_window, pair_view_candidate, siblings, stem_channels
    fmt = {"bf16": FOLD_BF16, "fp16": FOLD_F16, "fp32": FOLD_SPLIT3}[precision]
    f16 = precision == "fp16"
    chans, recs, checks = [], [], []
    n_coef = 0

    def at(name, shape=None):
        if name not in slots:
            raise KeyError(f"refold: the state has no entry {name}")
        o, numel, sh = slots[name]
        if shape is not None and tuple(sh) != tuple(shape):
            raise ValueError(f"refold: {name} has shape {tuple(sh)}, the engine's graph needs {tuple(shape)}")
        return o

    def bn(prefix, c, row0=0):
        return [at(f"{prefix}.{k}", (c,)) + row0 for k in BN_KEYS]

    def rec(dst, off, n, ds, layout, fmt_, wsrc=None, **kw):
        r = dict(dst=dst, off=off, n=tuple(n), ds=tuple(ds), layout=layout, fmt=fmt_, w=-1, w1=-1, coef=0, k=1, cin=1, r0=0, s0=0,
                 cout=0, flags=0, check=-1)
        if wsrc is not None:
            r.update(wsrc)
        r.update(kw)
        recs.append(r)
        return r

    def check_slot(name):
        if not f16:
            return -1
        checks.append(name)
        return len(checks) - 1

    wsrc_of = {}
    for i in packed_ops(g):
        op = g.ops[i]
        n = op.name
        if op.kind == "se":
            cr = op.cin // 4
            for key, name, shape in (("w1", ".conv1.weight", (cr, op.cin, 1, 1)), ("b1", ".conv1.bias", (cr,)),
                                     ("w2", ".conv2.weight", (op.cin, cr, 1, 1)), ("b2", ".conv2.bias", (op.cin,))):
                numel = 1
                for d in shape:
                    numel *= d
                rec((key, i), 0, (numel, 1, 1, 1), (1, 0, 0, 0), FOLD_COPY, FOLD_F32, w=at(n + name, shape))
            continue
        cout, k = op.cout, op.k
        ch = dict(bn=[[-1] * 4 for _ in range(3)], b=-1, coef=n_coef, n=cout)
        flags = 0
        if op.layout == "dp":
            cin_g = 1 if op.kind == "dw" else op.cin
            w = at(n + ".weight", (cout, cin_g, k, k))
            ch.update(layout=FOLD_C_DP, b=at(n + ".bias", (cout,)))
            ch["bn"][0] = bn(dp_bn(n), cout)
            wsrc = dict(layout=FOLD_W, w=w, k=k, cin=cin_g)
        elif op.layout == "rep":
            w = at(n + ".rbr_dense.conv.weight", (cout, op.cin, 3, 3))
            w1 = at(n + ".rbr_1x1.conv.weight", (cout, op.cin, 1, 1))
            ch["layout"] = FOLD_C_REP
            ch["bn"][0], ch["bn"][1] = bn(n + ".rbr_dense.bn", cout), bn(n + ".rbr_1x1.bn", cout)
            if n + ".rbr_identity.weight" in slots:
                ch["bn"][2] = bn(n + ".rbr_identity", cout)
                flags = FOLD_IDENTITY
            wsrc = dict(layout=FOLD_W_REP, w=w, w1=w1, k=3, cin=op.cin, flags=flags)
        elif op.layout == "qa":
            w = at(n + ".rbr_dense.conv.weight", (cout, op.cin, 3, 3))
            w1 = at(n + ".rbr_1x1.weight", (cout, op.cin, 1, 1))
            ch["layout"] = FOLD_C_QA
            ch["bn"][0], ch["bn"][1] = bn(n + ".rbr_dense.bn", cout), bn(n + ".bn", cout)
            flags = (FOLD_IDENTITY if op.identity else 0) | (FOLD_AVG if op.identity and op.avg else 0)
            wsrc = dict(layout=FOLD_W_QA, w=w, w1=w1, k=3, cin=op.cin, flags=flags)
        elif op.layout in ("cba", "cm"):
            cin_g = 1 if op.kind == "dw" else op.cin
            row0, rows = (op.w_row0, op.param_rows) if op.layout == "cm" else (0, cout)
            pre = n + (".block" if op.layout == "cba" else "")
            w = at(pre + ".conv.weight", (rows, cin_g, k, k)) + row0 * cin_g * k * k
            ch["layout"] = FOLD_C_BN
            ch["bn"][0] = bn(pre + ".bn", rows, row0)
            wsrc = dict(layout=FOLD_W, w=w, k=k, cin=cin_g)
        elif op.layout == "plain":
            w = at(n + ".weight", (cout, op.cin, k, k))
            ch.update(layout=FOLD_C_BIAS, b=at(n + ".bias", (cout,)))
            wsrc = dict(layout=FOLD_W_COPY, w=w, k=k, cin=op.cin)
        elif op.layout == "convT":
            w = at(n + ".upsample_transpose.weight", (op.cin, cout, 2, 2))
            ch.update(layout=FOLD_C_BIAS, b=at(n + ".upsample_transpose.bias", (cout,)))
            wsrc = dict(layout=FOLD_W_CONVT, w=w, k=2, cin=op.cin, cout=cout)
        else:
            raise ValueError(op.layout)
        chans.append(ch)
        wsrc["coef"] = ch["coef"]
        wsrc_of[i] = wsrc
        n_coef += 5 * cout
        bias1 = dict(wsrc, layout=FOLD_BIAS)
        if op.kind == "stem":        # w_dev[r][s][c][o], the pad channels stay zero
            cp = stem_channels(g, op)
            rec(("w_dev", i), 0, (cout, k, k, op.cin), (1, k * op.cin * cp, op.cin * cp, cp), wsrc["layout"], FOLD_F32, wsrc,
                check=check_slot(n))
            rec(("b_dev", i), 0, (cout, 1, 1, 1), (1, 0, 0, 0), FOLD_BIAS, FOLD_F32, bias1)
        elif op.kind == "dw":        # w_dev[r * k + s][c]
            rec(("w_dev", i), 0, (cout, k, k, 1), (1, k * cout, cout, 0), wsrc["layout"], FOLD_F32, wsrc)
            rec(("b_dev", i), 0, (cout, 1, 1, 1), (1, 0, 0, 0), FOLD_BIAS, FOLD_F32, bias1)
        elif op.kind == "convT":     # quadrant q = (dy, dx): [Cout][1][1][Cin] = w[:, :, dy, dx].t()
            for q in range(4):
                rec(("w", i, q), 0, (cout, 1, 1, op.cin), (op.cin, 0, 0, 1), FOLD_W_CONVT, fmt, wsrc, r0=q // 2, s0=q % 2,
                    check=check_slot(n))
            rec(("bias", i), 0, (cout, 1, 1, 1), (1, 0, 0, 0), FOLD_BIAS, FOLD_F32, bias1)
        else:                        # conv / pred: KRSC over the conv window
            lo, hi = conv_window(g, op)
            cw, c0 = hi - lo, op.src.c_off - lo
            rec(("w", i, 0), c0, (cout, k, k, op.cin), (k * k * cw, k * cw, cw, 1), wsrc["layout"], fmt, wsrc, check=check_slot(n))
            if pair_view_candidate(op):      # [Cout][3][2][2 * cw]: tap column 0 -> (0, cw + c), 1 -> (1, c), 2 -> (1, cw + c)
                for s0, off in ((0, cw + c0), (1, 2 * cw + c0), (2, 3 * cw + c0)):
                    rec(("w_pair", i), off, (cout, 3, 1, op.cin), (12 * cw, 4 * cw, 0, 1), wsrc["layout"], fmt, wsrc, s0=s0)
            rec(("bias", i), 0, (cout, 1, 1, 1), (1, 0, 0, 0), FOLD_BIAS, FOLD_F32, bias1)
    for i, j in siblings(g).items():     # [cls branch | reg branch] rows, unwindowed
        op = g.ops[i]
        k, cin, cout = op.k, op.cin, op.cout
        for half, o in enumerate((i, j)):
            ws = wsrc_of[o]
            rec(("w_fused", i), half * cout * k * k * cin, (cout, k, k, cin), (k * k * cin, k * cin, cin, 1), ws["layout"], fmt, ws)
            rec(("bias_fused", i), half * cout, (cout, 1, 1, 1), (1, 0, 0, 0), FOLD_BIAS, FOLD_F32, dict(ws, layout=FOLD_BIAS))
    return FoldPlan(chans, recs, checks, n_coef)


# ---------------------------------------------------------------------------------------------------- host replay
def _affine(flat, offs, c):
    g, b, m, v = (flat[o:o + c].double() for o in offs)
    scale = g / torch.sqrt(v + BN_EPS)
    return scale, b - m * scale


def host_coef(plan, flat):
    """The channel phase on the host: float64 [n_coef]."""
    coef = torch.zeros(plan.n_coef, dtype=torch.float64)
    for ch in plan.chans:
        c, L = ch["n"], ch["layout"]
        A, B, D, P = (torch.full((c,), v, dtype=torch.float64) for v in (1.0, 1.0, 0.0, 1.0))
        if L == FOLD_C_BIAS:
            bias = flat[ch["b"]:ch["b"] + c].double()
        else:
            s0, t0 = _affine(flat, ch["bn"][0], c)
            A = s0
            if L == FOLD_C_DP:
                bias = flat[ch["b"]:ch["b"] + c].double() * s0 + t0
            elif L == FOLD_C_BN:
                bias = t0
            elif L == FOLD_C_QA:
                s1, t1 = _affine(flat, ch["bn"][1], c)
                P, bias = s1, t0 * s1 + t1
            else:
                s1, t1 = _affine(flat, ch["bn"][1], c)
                B, bias = s1, t0 + t1
                if ch["bn"][2][0] >= 0:
                    s2, t2 = _affine(flat, ch["bn"][2], c)
                    D, bias = s2, bias + t2
        coef[ch["coef"]:ch["coef"] + 5 * c] = torch.stack([A, B, D, P, bias], 1).reshape(-1)
    return coef


def host_values(r, flat, coef, cache=None):
    """The float64 values of one record, shaped as its domain (o, r, s, c).  `cache` keeps the op-level weight a record slices
    (the column-pair view and sibling records reuse it)."""
    n, L = r["n"], r["layout"]
    o = n[0]
    cf = coef[r["coef"]:r["coef"] + 5 * o].view(o, 5)
    if L == FOLD_BIAS:
        return cf[:, 4].reshape(o, 1, 1, 1)
    if L == FOLD_COPY:
        return flat[r["w"]:r["w"] + o].double().reshape(o, 1, 1, 1)
    if L == FOLD_W_CONVT:
        cin, cout = n[3], r["cout"]
        w = flat[r["w"]:r["w"] + cin * cout * 4].view(cin, cout, 2, 2)[:, :, r["r0"], r["s0"]]
        return w.t().double().reshape(o, 1, 1, cin)
    key = (r["w"], L, r["coef"])
    v = cache.get(key) if cache is not None else None
    if v is None:
        k, cin = r["k"], r["cin"]
        w = flat[r["w"]:r["w"] + o * cin * k * k].view(o, cin, k, k).double().permute(0, 2, 3, 1)     # (o, r, s, c)
        A = cf[:, 0].reshape(o, 1, 1, 1)
        if L == FOLD_W_COPY:
            v = w
        elif L == FOLD_W:
            v = w * A
        else:
            w1 = flat[r["w1"]:r["w1"] + o * cin].view(o, cin).double()
            pad = torch.zeros(o, 3, 3, cin, dtype=torch.float64)
            pad[:, 1, 1, :] = w1 * cf[:, 1:2] if L == FOLD_W_REP else w1
            v = w * A + pad                 # the off-centre taps add +0.0, as fold.py's pad(k1) / pad(W1)
            idx = torch.arange(cin)
            if L == FOLD_W_REP:
                if r["flags"] & FOLD_IDENTITY:
                    v[idx, 1, 1, idx] += cf[:, 2]
            else:
                if r["flags"] & FOLD_IDENTITY:
                    v[idx, 1, 1, idx] += 1.0
                if r["flags"] & FOLD_AVG:
                    v[idx, :, :, idx] += 1.0 / 9.0
                v = v * cf[:, 3].reshape(o, 1, 1, 1)
        if cache is not None:
            cache[key] = v
    return v[:, r["r0"]:r["r0"] + n[1], r["s0"]:r["s0"] + n[2], :n[3]]


def host_check(plan, flat, coef):
    """The fp16 range check of a plan on the host: raises fold.to_f16's ValueError for the first failing slot."""
    cache = {}
    for r in plan.recs:
        if r["check"] >= 0:
            v = host_values(r, flat, coef, cache)
            if not torch.isfinite(v.float().to(torch.float16)).all():
                raise f16_range_error(plan.checks[r["check"]], float(v.abs().max()))


def replay_host(plan, flat, resolve):
    """Execute the plan's records with torch's float64 CPU ops: the fp16 check (raising before anything is written), then
    every record into resolve(dst key) (a contiguous CPU tensor)."""
    flat = flat.cpu()
    coef = host_coef(plan, flat)
    if plan.checks:
        host_check(plan, flat, coef)
    cache = {}
    for r in plan.recs:
        t = resolve(r["dst"])
        f = host_values(r, flat, coef, cache).float()
        d = t.view(-1)
        if r["fmt"] == FOLD_SPLIT3:
            for q, p in enumerate(ops.split3(f)):
                d.as_strided(r["n"], r["ds"], d.storage_offset() + r["off"] + q * t[0].numel()).copy_(p)
            continue
        cast = {FOLD_F32: torch.float32, FOLD_BF16: torch.bfloat16, FOLD_F16: torch.float16}[r["fmt"]]
        d.as_strided(r["n"], r["ds"], d.storage_offset() + r["off"]).copy_(f.to(cast))


# ---------------------------------------------------------------------------------------------------- device tables
def device_tables(plan, resolve, device):
    """(chans, recs, n_blocks, coef, checks) of a plan on the device; records point at resolve(dst key)."""
    chans = (FoldChan * max(len(plan.chans), 1))()
    for a, ch in zip(chans, plan.chans):
        for b in range(3):
            for q in range(4):
                a.bn[b][q] = ch["bn"][b][q]
        a.b, a.coef, a.layout, a.n = ch["b"], ch["coef"], ch["layout"], ch["n"]
    recs = [r for r in plan.recs if r["n"][0] * r["n"][1] * r["n"][2] * r["n"][3] > 0]
    arr = (FoldRec * max(len(recs), 1))()
    blk = 0
    for a, r in zip(arr, recs):
        t = resolve(r["dst"])
        a.dst = t.data_ptr() + r["off"] * t.element_size()
        a.plane_stride = t[0].numel() if r["fmt"] == FOLD_SPLIT3 else 0
        for q in range(4):
            a.ds[q], a.n[q] = r["ds"][q], r["n"][q]
        for key in ("w", "w1", "coef", "layout", "fmt", "k", "cin", "r0", "s0", "cout", "flags", "check"):
            setattr(a, key, r[key])
        a.blk0 = blk
        blk += -(-(r["n"][0] * r["n"][1] * r["n"][2] * r["n"][3]) // FOLD_CHUNK)
    as_dev = lambda a: torch.frombuffer(bytearray(bytes(a)), dtype=torch.uint8).to(device)
    return dict(chans=as_dev(chans), n_chans=len(plan.chans), recs=as_dev(arr), n_recs=len(recs), n_blocks=blk,
                coef=torch.empty(max(plan.n_coef, 1), dtype=torch.float64, device=device),
                checks=torch.zeros(2 * max(len(plan.checks), 1), dtype=torch.int64, device=device))


def launch(lib, h, tables, flat, check_only, stream):
    t = tables
    _lib.check(lib.yv6_fold(h, flat.data_ptr(), t["chans"].data_ptr(), t["n_chans"], t["recs"].data_ptr(), t["n_recs"],
                            t["n_blocks"], t["coef"].data_ptr(), t["checks"].data_ptr(), int(check_only), _lib.stream_ptr(stream)))


def device_check(lib, h, plan, tables, flat, stream):
    """The fp16 range check on the device (one host sync): raises fold.to_f16's ValueError for the first failing slot."""
    if not plan.checks:
        return
    with torch.cuda.stream(stream):
        tables["checks"].zero_()
        launch(lib, h, tables, flat, True, stream)
        res = tables["checks"].cpu().view(-1, 2)
    for slot in range(len(plan.checks)):
        if int(res[slot, 0]):
            wmax = C.c_double.from_buffer_copy(C.c_uint64(int(res[slot, 1]) & (2 ** 64 - 1))).value
            raise f16_range_error(plan.checks[slot], wmax)
