"""The launches of the self-distillation step run alone through the C ABI and checked against float64 at the distillation
shapes: every yv6_kl_rows launch of ComputeLoss[NS].distill_forward_backward, the teacher's forward-only engine, and the
injection of the channel-wise term's neck-output gradients.

Part 1, yv6_kl_rows.  The N / S recipe (tools/bench_distill.py: YOLOv6-S, 640, batch 32, nc 80, A = 8400, T = 20) and the
M / L recipe (M, 640, batch 8), each with its three terms exactly as the step passes them:
  class: rows B*A, C = 80, T = 20, no mask, scale = T^2 (loss weights and decay 1);
  DFL: rows 4*B*A, C = 17, mask = fg (uint8 per anchor, 4 rows per entry), count = out[5] (num_pos, mean over 4 num_pos
    rows), gate = out[4] (target_scores_sum, the term is 0 unless it is > 0);
  channel-wise: one launch per neck level, rows = images x channels, C = H*W (6400 / 1600 / 400 at 640), T = 1,
    scale = 10 / (N C).
And edges: C in {1, 31, 32, 33} (a warp's lanes over the row), rows in {1, 7, 9} and one more row than the grid has warps
(8 x 8 x SMs: exactly one warp takes a second row), C = 25600 (the first neck level of a 1280-px L6), an all-zero mask,
num_pos = 0, target_scores_sum = 0, rows where student == teacher, and a row dominated by one position 80 above the rest
at T = 1.  Inputs look like the step's: post-sigmoid scores with the student a perturbation of the teacher in logit space,
DFL logits ~ N(0, 3), bf16-representable SiLU-like neck activations.  The gradient buffer holds a random prior (the kernel
adds to it) of the size of the term, the accumulator a random prior, and guard elements on both sides of each hold 2^100.
Every class and DFL launch at the training shapes takes the kernel's grid-stride loop over rows: rows > 8 x blocks, with
blocks = min(ceil(rows / 8), 8 x SMs) as yv6_kl_rows computes it (asserted).  The channel-wise launches at these shapes have
at most one row per warp; the edge with one row more than warps runs the loop at C = 6400.

References, in float64 from the fp32 operands, with iT = fp32(1 / T) as the kernel scales (not 1 / T): per row
log p = log_softmax(s iT), log q = log_softmax(t iT), KL = sum q (log q - log p); eff = scale, divided by the active row
count when a count is given, and 0 when the count is 0 or the gate is not > 0.
  value: acc - prior against eff sum_active KL.  The kernel works in double: per row the two log-sum-exps carry a relative
    error of (C/32 + 7) u from a lane's sum of C/32 exponentials, the 5-level shuffle tree and exp / log (u = 2^-53), which
    enters every log-probability as an absolute error; each log-probability is also rounded relative to |s iT| + |lse|; the
    KL sum over C/32 terms per lane plus the tree adds (C/32 + 5) u of sum q |log q - log p|.  All of it is below
    K_C u (1 + S_row), S_row = sum q (|log p| + |log q|), with K_C = 64 + C/16 (69 at C = 80, 65 at 17, 464 at 6400).  The
    row sums are then added per warp (n_w rows), by a shuffle tree and an 8-warp block sum, then by one atomic add per block
    onto the prior: (n_w + 13 + blocks) u sum |KL| plus (blocks + 2) u (|prior| + |acc|) for the additions onto the prior and
    the subtraction of the check.  Per row the bar is ~1e-14 of S_row, ~1e8 below the KL of a row of these inputs; summed
    over all rows it stays below the smallest single active row's term (asserted for every launch at the training shapes:
    a dropped or doubled row is seen in the value alone).
  gradient: each active element against prior + eff (p - q) iT; one fp32 rounding of the term and one of the fp32 add,
    2^-24 (|term| + |prior + term|), plus the float64 term's own error, K_C u eff iT (p + q) (which also covers the
    second-order u^2 |term| of bounding the add by the exact term), plus 2^-149 for a rounding in fp32's subnormal range.
    Two roundings that each come close to half an ulp put an element near the bar (ratios ~0.999 over millions of
    elements); a lost or doubled term is off by the whole term, a 1/T slip by 19 terms at T = 20.
  inactive elements (masked rows; every element when eff = 0) keep their prior bit for bit, and so do the accumulator when
    eff = 0, the guard elements and the inputs.
The kernel's iT = fp32(1/T) differs from 1/T by |fp32(1/T) T - 1| <= 2^-24 (asserted on its own), ~2^-22 relative on the KL
at T = 20: the reference uses the kernel's iT instead of widening the bar.

Part 2, the teacher's forward.  Model.teacher_engine() of the N / S recipe's teacher (S with the DFL head, reg_max 16,
fuse_ab, planned at 640, batch 32, uint8) and of an M teacher (640, batch 2).  After begin_step every packed forward weight
equals bf16 of its master parameter in KRSC order (the stem's fp32 [r][s][c][Cout]) and every packed bias its fp32 master
padded with zeros, bit for bit.  Every distinct forward launch record runs alone under the training-forward checks of
tests/test_gpu_forward_launches.py (conv, stats, apply, pool; the uint8 stem against float64 of the fp32 product
u8 x in_scale).  Every statistics descriptor carries null running statistics, the plan has no anchor-aided pred conv and
no pack launch, and the whole flat parameter buffer (running statistics and num_batches_tracked included) is bit-identical
after a full forward.

Part 3, injection.  With external neck-output gradients, backward(first=0, last=0) runs no launch: afterwards each neck
slice holds bf16 of the injected NCHW gradient in NHWC, bit for bit, and every other element of every gradient buffer is
what the clears of zero_gbufs left (zero) or the 2^100 it held.

Each test prints its distinct / total launches, worst error / bar per kind and the time taken."""
import ctypes as C
import math
import time
import types

import numpy as np
import pytest
import torch

import test_gpu_backward_launches as bwd
import test_gpu_forward_launches as fwd

pytestmark = pytest.mark.gpu

F32, F64, BF16 = torch.float32, torch.float64, torch.bfloat16
U64, U32 = 2.0 ** -53, 2.0 ** -24
SENT = 2.0 ** 100
GUARD = 32                 # sentinel elements on each side of the gradient and the accumulator
NC, T_DISTILL, REG = 80, 20.0, 17
CWD = 10.0                 # loss_weight['cwd']


# ---------------------------------------------------------------------------------------------------------------- yv6_kl_rows
def inv_t(T):
    """The kernel's 1.f / temperature in fp32, as a double."""
    return float(np.float32(1.0) / np.float32(T))


def kl_blocks(rows, sms):
    """yv6_kl_rows's grid: min(ceil(rows / 8), 8 x SMs) blocks of 8 warps."""
    return min((rows + 7) // 8, 8 * sms)


def kl_case(name, s, t, T, scale, mask=None, rpm=1, num_pos=None, tss=None):
    rows, Cc = s.shape
    return types.SimpleNamespace(name=name, s=s.contiguous(), t=t.contiguous(), rows=rows, C=Cc, T=float(T), iT=inv_t(T),
                                 scale=float(scale), mask=mask, rpm=rpm, num_pos=num_pos, tss=tss)


def kl_expected(c, sms):
    """float64 reference of one launch: eff, active rows, per-row KL and S_row, the gradient term, p + q, and the grid."""
    eff = c.scale
    if c.num_pos is not None:
        n = float(c.num_pos) * c.rpm
        eff = c.scale / n if n > 0 else 0.0
    if c.tss is not None and not float(c.tss) > 0:
        eff = 0.0
    if c.mask is None:
        active = torch.ones(c.rows, dtype=torch.bool, device=c.s.device)
    else:
        active = c.mask.reshape(-1).repeat_interleave(c.rpm)[:c.rows] != 0
    a = torch.log_softmax(c.s.double() * c.iT, -1)
    b = torch.log_softmax(c.t.double() * c.iT, -1)
    p, q = a.exp(), b.exp()
    kl = (q * (b - a)).sum(-1)
    S = (q * (a.abs() + b.abs())).sum(-1)
    blocks = kl_blocks(c.rows, sms)
    return types.SimpleNamespace(eff=eff, active=active, kl=kl, S=S, term=eff * (p - q) * c.iT, pq=p + q, blocks=blocks,
                                 per_warp=-(-c.rows // (8 * blocks)), K=64 + c.C / 16)


def kl_value_ratio(c, e, acc0, acc):
    """|(acc - prior) - eff sum KL| / bar, and the bar over the smallest positive active row term (module docstring)."""
    got = float(acc) - float(acc0)
    kl, S = e.kl[e.active], e.S[e.active]
    want = e.eff * float(kl.sum())
    bar = (abs(e.eff) * U64 * (e.K * float((1 + S).sum()) + (e.per_warp + 13 + e.blocks) * float(kl.abs().sum()))
           + (e.blocks + 2) * U64 * (abs(float(acc0)) + abs(float(acc))))
    pos = kl[kl > 0]
    smallest = abs(e.eff) * float(pos.min()) if pos.numel() else math.inf
    return abs(got - want) / bar, bar / smallest


def kl_grad_ratio(c, e, g0, g):
    """Active elements against prior + eff (p - q) iT: 2^-24 (|term| + |prior + term|) + K_C u eff iT (p + q)."""
    a = e.active
    ref = g0[a].double() + e.term[a]
    bar = U32 * (e.term[a].abs() + ref.abs()) + e.K * U64 * abs(e.eff) * c.iT * e.pq[a] + 2.0 ** -149
    return bwd.ratio(g[a], ref, bar)


def assert_untouched(c, e, g0, g, what):
    """Masked-out rows (every row when eff = 0) keep their prior bit for bit."""
    keep = ~e.active if e.eff != 0 else torch.ones_like(e.active)
    bad = keep & (g.view(torch.int32) != g0.view(torch.int32)).any(-1)
    if bool(bad.any()):
        raise AssertionError(f"{what}: {int(bad.sum())} inactive rows changed, first row {int(bad.nonzero()[0, 0])}")


def kl_buffers(c, e, gen):
    """The launch's gradient (a prior of the size of the term: the fp32 add then rounds at the term's scale) and accumulator
    (a N(0, 1) prior), each between guards of 2^100, and the loss-output vector holding num_pos and target_scores_sum."""
    dev = c.s.device
    mag = float(e.term[e.active].abs().mean()) if bool(e.active.any()) and e.eff != 0 else 1.0
    gbuf = torch.full((c.rows * c.C + 2 * GUARD,), SENT, dtype=F32, device=dev)
    g = gbuf[GUARD:GUARD + c.rows * c.C].view(c.rows, c.C)
    g.copy_(torch.randn(c.rows, c.C, generator=gen, device=dev) * (mag if mag > 0 else 1.0))
    abuf = torch.full((2 * GUARD + 1,), SENT, dtype=F64, device=dev)
    abuf[GUARD] = torch.randn(1, generator=gen, device=dev, dtype=F64)[0]
    out = torch.full((8,), SENT, dtype=F64, device=dev)
    count = gate = 0
    if c.num_pos is not None:
        out[5] = float(c.num_pos)
        count = out.data_ptr() + 5 * 8
    if c.tss is not None:
        out[4] = float(c.tss)
        gate = out.data_ptr() + 4 * 8
    return g, gbuf, abuf, out, count, gate


def checked_kl(c, sms, gen):
    """Run one launch with the step's arguments and check it; returns (value ratio, gradient ratio, summed value bar / smallest
    row term, the reference)."""
    from yolov6_b200 import _lib
    lib, h, sp = _lib.lib(), _lib.handle(0), _lib.stream_ptr()
    e = kl_expected(c, sms)
    g, gbuf, abuf, out, count, gate = kl_buffers(c, e, gen)
    g0, acc0, s0, t0, out0 = g.clone(), abuf[GUARD].clone(), c.s.clone(), c.t.clone(), out.clone()
    mask = c.mask.data_ptr() if c.mask is not None else 0
    bwd.check(lib.yv6_kl_rows(h, c.s.data_ptr(), c.t.data_ptr(), c.rows, c.C, c.T, mask, c.rpm, c.scale, count, gate,
                              abuf.data_ptr() + GUARD * 8, g.data_ptr(), sp), lib)
    torch.cuda.synchronize()
    acc = abuf[GUARD].clone()
    assert (gbuf[:GUARD] == SENT).all() and (gbuf[-GUARD:] == SENT).all(), f"{c.name}: wrote outside the gradient"
    assert (abuf[:GUARD] == SENT).all() and (abuf[GUARD + 1:] == SENT).all(), f"{c.name}: wrote outside the accumulator"
    assert torch.equal(c.s, s0) and torch.equal(c.t, t0) and torch.equal(out, out0), f"{c.name}: changed an input"
    assert_untouched(c, e, g0, g, c.name)
    if e.eff == 0:
        assert acc.view(torch.int64).item() == acc0.view(torch.int64).item(), f"{c.name}: accumulator changed with eff = 0"
        return 0.0, 0.0, 0.0, e
    rv, rel = kl_value_ratio(c, e, acc0, acc)
    rg = kl_grad_ratio(c, e, g0, g)
    assert rv <= 1.0, f"{c.name}: value error {rv:.3f} x the bar"
    assert rg <= 1.0, f"{c.name}: gradient error {rg:.3f} x the bar"
    return rv, rg, rel, e


def scores_pair(gen, rows, nc, dev):
    """Teacher post-sigmoid scores and a student perturbed in logit space, both in (0, 1)."""
    z = torch.randn(rows, nc, generator=gen, device=dev) * 2.0 - 2.0
    t = torch.sigmoid(z)
    s = torch.sigmoid(z + torch.randn(rows, nc, generator=gen, device=dev) * 0.5)
    return s.float().contiguous(), t.float().contiguous()


def dfl_pair(gen, rows, dev):
    t = torch.randn(rows, REG, generator=gen, device=dev) * 3.0
    return (t + torch.randn(rows, REG, generator=gen, device=dev) * 0.5).contiguous(), t.contiguous()


def neck_pair(gen, rows, C, dev):
    """bf16-representable SiLU-like activations: silu of N(0, 1.5), rounded to bf16; the student a perturbation."""
    z = torch.randn(rows, C, generator=gen, device=dev) * 1.5
    t = torch.nn.functional.silu(z).to(BF16).float()
    s = torch.nn.functional.silu(z + torch.randn(rows, C, generator=gen, device=dev) * 0.3).to(BF16).float()
    return s.contiguous(), t.contiguous()


def fg_mask(gen, B, A, dev, frac=0.03):
    return (torch.rand(B, A, generator=gen, device=dev) < frac).to(torch.uint8).contiguous()


def neck_shapes(cfg, size):
    """(channels, H*W) of the three neck levels the channel-wise term reads."""
    from yolov6_b200.model import build_model
    g = build_model(cfg, NC, torch.device("cpu")).graph
    return [(t.c, (size >> g.bufs[t.buf].level) ** 2) for t in g.feat[:3]]


RECIPES = {"ns_s640_b32": ("yolov6s", 640, 32), "ml_m640_b8": ("yolov6m", 640, 8)}


def recipe_cases(name, gen, dev):
    cfg, size, B = RECIPES[name]
    A = sum((size // s) ** 2 for s in (8, 16, 32))
    assert A == 8400
    T = T_DISTILL
    s, t = scores_pair(gen, B * A, NC, dev)
    yield kl_case(f"{name} class", s, t, T, T * T), True
    del s, t
    fg = fg_mask(gen, B, A, dev)
    s, t = dfl_pair(gen, B * A * 4, dev)
    yield kl_case(f"{name} dfl", s, t, T, T * T, mask=fg, rpm=4, num_pos=int(fg.sum()), tss=17.25), True
    del s, t
    for ch, hw in neck_shapes(cfg, size):
        s, t = neck_pair(gen, B * ch, hw, dev)
        yield kl_case(f"{name} cw C={hw}", s, t, 1.0, CWD / (B * ch)), False


def test_kl_rows_scales_by_the_fp32_reciprocal_of_t():
    """The kernel's iT = fp32(1/T) against the exact 1/T: within 2^-24 relative, ~2^-22 on the KL at T = 20 (KL ~ iT^2)."""
    for T in (1.0, 20.0, 3.0, 7.0):
        d = abs(inv_t(T) * T - 1.0)
        assert d <= 2.0 ** -24, (T, d)
    assert inv_t(1.0) == 1.0 and inv_t(T_DISTILL) != 1.0 / T_DISTILL


@pytest.mark.parametrize("recipe", list(RECIPES))
def test_kl_rows_launches_at_the_distillation_shapes(recipe):
    t0 = time.time()
    sms = bwd.num_sms()
    gen = torch.Generator(device="cuda").manual_seed(20261017)
    worst, rels, n = {"value": 0.0, "grad": 0.0}, [], 0
    for c, strided in recipe_cases(recipe, gen, torch.device("cuda")):
        rv, rg, rel, e = checked_kl(c, sms, gen)
        n += 1
        if strided:
            assert c.rows > 8 * e.blocks, f"{c.name}: {c.rows} rows fit one per warp of {e.blocks} blocks (no grid-stride loop)"
        assert rel < 1.0, f"{c.name}: the summed value bar is {rel:.2g} of the smallest row's term"
        worst["value"], worst["grad"] = max(worst["value"], rv), max(worst["grad"], rg)
        rels.append(f"{c.name} {rel:.1e} ({c.rows} rows, {e.per_warp}/warp)")
        del c, e
        torch.cuda.empty_cache()
    print(f"\n{recipe}: kl_rows launches checked {n}/{n}; worst error / bar: value {worst['value']:.3f}, gradient "
          f"{worst['grad']:.3f}; summed value bar / smallest row term: " + ", ".join(rels) + f"; {time.time() - t0:.1f} s")


def edge_cases(gen, dev, sms):
    warps = 8 * 8 * sms
    for Cc in (1, 31, 32, 33):
        s, t = neck_pair(gen, 300, Cc, dev)
        yield kl_case(f"C={Cc}", s, t, 1.0, 0.7)
        s, t = scores_pair(gen, 300, Cc, dev)
        yield kl_case(f"C={Cc} T=20", s, t, T_DISTILL, 400.0)
    for r in (1, 7, 9):
        s, t = scores_pair(gen, r, NC, dev)
        yield kl_case(f"rows={r}", s, t, T_DISTILL, 400.0)
    s, t = scores_pair(gen, warps + 1, NC, dev)
    yield kl_case(f"rows={warps + 1} (warps + 1)", s, t, T_DISTILL, 400.0)
    s, t = neck_pair(gen, warps + 1, 6400, dev)
    yield kl_case(f"rows={warps + 1} C=6400", s, t, 1.0, CWD / (warps + 1))
    s, t = neck_pair(gen, 2 * 128, 25600, dev)
    yield kl_case("C=25600 (L6 at 1280)", s, t, 1.0, CWD / 256)
    B, A = 4, 8400
    s, t = dfl_pair(gen, B * A * 4, dev)
    zero = torch.zeros(B, A, dtype=torch.uint8, device=dev)
    yield kl_case("dfl all-zero mask", s, t, T_DISTILL, 400.0, mask=zero, rpm=4, num_pos=0, tss=3.5)
    fg = fg_mask(gen, B, A, dev)
    yield kl_case("dfl num_pos = 0", s, t, T_DISTILL, 400.0, mask=fg, rpm=4, num_pos=0, tss=3.5)
    yield kl_case("dfl target_scores_sum = 0", s, t, T_DISTILL, 400.0, mask=fg, rpm=4, num_pos=int(fg.sum()), tss=0.0)
    yield kl_case("dfl mask with 0xff entries", s, t, T_DISTILL, 400.0, mask=fg * 255, rpm=4, num_pos=int(fg.sum()), tss=3.5)
    s, t = scores_pair(gen, 4096, NC, dev)
    s[::3] = t[::3]
    yield kl_case("student == teacher on every third row", s, t, T_DISTILL, 400.0)
    s, t = neck_pair(gen, 64, 400, dev)
    s[:, 17] += 80.0
    t[5, 203] += 80.0
    t[9, 17] += 80.0
    yield kl_case("one position 80 above the rest, T = 1", s, t, 1.0, 1.0)


def test_kl_rows_edges():
    t0 = time.time()
    sms = bwd.num_sms()
    gen = torch.Generator(device="cuda").manual_seed(20261018)
    worst, n = {"value": 0.0, "grad": 0.0}, 0
    for c in edge_cases(gen, torch.device("cuda"), sms):
        rv, rg, _, e = checked_kl(c, sms, gen)
        n += 1
        worst["value"], worst["grad"] = max(worst["value"], rv), max(worst["grad"], rg)
        if "student == teacher" in c.name:      # identical rows: p = q exactly, the gradient keeps its prior bit for bit
            g_rows = torch.zeros(c.rows, dtype=torch.bool, device=c.s.device)
            g_rows[::3] = True
            assert bool((e.kl[g_rows] == 0).all())
        if "warps + 1" in c.name or "C=6400" in c.name:
            assert c.rows > 8 * e.blocks
    print(f"\nkl_rows edges: launches checked {n}/{n}; worst error / bar: value {worst['value']:.3f}, gradient "
          f"{worst['grad']:.3f}; {time.time() - t0:.1f} s")


# ---------------------------------------------------------------------------------------------------------------- the teacher
TEACHERS = {
    "yolov6s_dfl_fuse_ab_640_b32_u8": dict(cfg="yolov6s", size=640, batch=32, u8=True, fuse_ab=True, dfl=True),
    "yolov6m_640_b2": dict(cfg="yolov6m", size=640, batch=2),
}


def teacher_of(name):
    c = TEACHERS[name]
    dev = torch.device("cuda:0")
    m = bwd.seeded_model(c["cfg"], dev, fuse_ab=c.get("fuse_ab", False), dfl=c.get("dfl", False)).train()
    eng = m.teacher_engine()
    eng._plan(c["batch"], c["size"], c["size"], torch.uint8 if c.get("u8") else F32)
    return m, eng


def teacher_mem(eng):
    """A teacher has no gradient buffers, scratch or gradient heads: its activations, statistics, heads, input, branch
    outputs, packed weights and the flat parameters."""
    named = [("buf", t) for t in eng.bufs] + [("arena", eng.zero_arena)] + [("stat", t) for t in eng.stat_out.values()]
    named += [("head", eng.cls), ("head", eng.reg), ("img", eng.x_static), ("param", eng.flat.pflat)]
    named += [("raw", br["x"]) for ctx in eng.ctx if ctx and "branches" in ctx for br in ctx["branches"] if br["k"]]
    named += [("qa_t", ctx["t"]) for ctx in eng.ctx if ctx and "t" in ctx]
    mem = bwd.Mem(named)
    for t in packed_tensors(eng.wts):
        mem.ts.append((t.data_ptr(), t.data_ptr() + t.numel() * t.element_size(), "w", t))
    return mem


def packed_tensors(v):
    if torch.is_tensor(v):
        yield v
    elif isinstance(v, dict):
        for u in v.values():
            yield from packed_tensors(u)
    elif isinstance(v, (list, tuple)):
        for u in v:
            yield from packed_tensors(u)


def check_pack(m, eng):
    """Every packed forward weight against its master parameter, bit for bit; returns the number of tensors compared."""
    from yolov6_b200.train import conv_weight_name, op_branches
    P = dict(m.named_parameters())
    n = 0

    def same(got, want, what):
        nonlocal n
        assert got.dtype == want.dtype and got.shape == want.shape, f"{what}: {got.dtype} {tuple(got.shape)}"
        iv = torch.int16 if got.dtype == BF16 else torch.int32
        assert torch.equal(got.contiguous().view(iv), want.contiguous().view(iv)), f"{what}: packed weight differs"
        n += 1

    def bias(got, want, what):
        assert not bool(got[want.numel():].any()), f"{what}: bias padding"
        same(got[:want.numel()], want.detach().float(), what)

    for i, W in eng.wts.items():
        op = eng.g.ops[i]
        if op.kind == "pred":
            w = P[op.name + ".weight"].detach()
            same(W["w"], w.reshape(op.cout, op.cin).to(BF16).reshape(op.cout, 1, 1, op.cin), op.name)
            bias(W["bias"], P[op.name + ".bias"], op.name + " bias")
        elif op.kind == "convT":
            w = P[op.name + ".upsample_transpose.weight"].detach()            # [Cin][Cout][2][2]
            for q in range(4):
                same(W["w"][q], w[:, :, q // 2, q % 2].t().to(BF16).reshape(op.cout, 1, 1, op.cin), f"{op.name} quadrant {q}")
            bias(W["bias"], P[op.name + ".upsample_transpose.bias"], op.name + " bias")
        else:
            for ent, (prefix, k) in zip(W["br"], op_branches(op)):
                if k == 0:
                    continue
                w = P[conv_weight_name(op, prefix)].detach()[op.w_row0:op.w_row0 + op.cout]      # [Cout][Cin][k][k]
                if op.kind == "stem":
                    want = torch.zeros(3, 3, 3, op.cout, dtype=F32, device=w.device)
                    if k == 3:
                        want[:] = w.permute(2, 3, 1, 0)
                    else:
                        want[1, 1] = w[:, :, 0, 0].t()
                    same(ent["w"], want, f"{op.name}{prefix} stem")
                else:
                    same(ent["w"], w.permute(0, 2, 3, 1).to(BF16), f"{op.name}{prefix}")
    return n


def tcheck_stem_any(lib, h, sp, mem, eng, c, gen):
    """The fp32-math stem; with a uint8 input against float64 of the fp32 products u8 x in_scale."""
    d = c.desc
    if eng.x_static.dtype != torch.uint8:
        return fwd.tcheck_stem(lib, h, sp, mem, eng, c, gen)
    assert d.fp32_math == 1 and d.x == eng.x_static.data_ptr()
    x = eng.x_static
    x.copy_(torch.randint(0, 256, x.shape, generator=gen, device=x.device, dtype=torch.uint8))
    xf = x.float() * torch.tensor(d.in_scale, dtype=F32, device=x.device)
    N, H, W, Cout = d.N, d.H, d.W, d.Cout
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    w = mem.at(d.w, F32, (3, 3, 3, Cout)).permute(3, 0, 1, 2)
    b = mem.at(d.bias, F32, (Cout,)) if d.bias else torch.zeros(Cout, dtype=F32, device=w.device)
    yv = mem.at(d.y, BF16, (N, Ho, Wo, Cout))
    got, = fwd.guarded(mem, [yv], lambda: bwd.check(lib.yv6_stem_fwd(h, C.byref(d), sp), lib))
    ref, R, z = fwd.conv_ref(xf.permute(0, 2, 3, 1), w, b, 2, 1, d.act)
    return bwd.ratio(got, ref, fwd.out_bar(ref, R, z, d.act, bf16_out=True, planes3=False, fast_silu=False))


TEACHER_KINDS = ("stem", "conv", "stats", "apply", "qa", "pool")


@pytest.mark.parametrize("name", list(TEACHERS))
def test_teacher_forward_launches(name):
    from yolov6_b200 import _lib
    t0 = time.time()
    m, eng = teacher_of(name)
    lib, h, sp = eng.lib, eng.h, _lib.stream_ptr()
    fl = eng.flat
    flat0 = [t.clone() for t in (fl.pflat, fl.iflat)]
    eng.begin_step()
    torch.cuda.synchronize()
    packed = check_pack(m, eng)
    # a full forward leaves every running statistic and counter of the teacher's model as it was
    x = eng.x_static
    x.copy_(torch.randint(0, 256, x.shape, device=x.device, dtype=torch.uint8) if x.dtype == torch.uint8 else torch.rand(x.shape, device=x.device))
    eng.run_forward(sp)
    torch.cuda.synchronize()
    for a, b in zip(flat0, (fl.pflat, fl.iflat)):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), f"{name}: the teacher's forward changed its flat state"
    assert not any(c.fn == "yv6_head_ab_pack" for c in eng.fwd_calls) and not hasattr(eng, "_ab"), "anchor-aided branch planned"
    mem = teacher_mem(eng)
    for c in eng.fwd_calls:
        if c.kind == "conv":
            assert mem.find(c.desc.y)[0] in ("buf", "raw", "head"), f"{name}: a conv writes outside the teacher's outputs"
        if c.kind == "stats":
            d = c.desc
            assert all(d.running_mean[b] in (0, None) and d.running_var[b] in (0, None) for b in range(3)), \
                f"{name}: a statistics launch carries running statistics"
        if c.kind == "qa":
            assert not c.desc.running_mean and not c.desc.running_var
    gen = torch.Generator(device="cuda").manual_seed(20261019)
    worst = {k: 0.0 for k in TEACHER_KINDS}
    seen = {k: set() for k in TEACHER_KINDS}
    total = {k: 0 for k in TEACHER_KINDS}
    for c in eng.fwd_calls:
        k = c.kind
        assert k in TEACHER_KINDS, k
        total[k] += 1
        sig = bwd.signature(c.desc, mem) if c.desc is not None else tuple(
            (mem.find(a)[0], mem.find(a)[2]) if isinstance(a, int) and a > 1 << 20 and mem.find(a) else
            (tuple(a) if isinstance(a, C.Array) else a) for a in c.args)
        if sig in seen[k]:
            continue
        seen[k].add(sig)
        r = {"conv": lambda: fwd.tcheck_conv(lib, h, sp, mem, c, gen), "stem": lambda: tcheck_stem_any(lib, h, sp, mem, eng, c, gen),
             "stats": lambda: fwd.tcheck_stats(lib, h, sp, mem, eng, c, gen), "apply": lambda: fwd.tcheck_apply(lib, h, sp, mem, c, gen),
             "qa": lambda: fwd.tcheck_qa(lib, h, sp, mem, eng, c, gen), "pool": lambda: fwd.tcheck_pool(lib, h, sp, mem, c, gen)}[k]()
        assert r <= 1.0, f"{name}: {k} launch {len(seen[k])}: error {r:.3f} x the bar"
        worst[k] = max(worst[k], r)
    # the checks only read the flat parameters (gamma, beta, shortcut alpha): no teacher launch wrote them
    assert torch.equal(flat0[0].view(torch.uint8), fl.pflat.view(torch.uint8)), f"{name}: a teacher launch wrote the flat parameters"
    print(f"\n{name} (teacher forward): packed weights bit-exact {packed}; distinct launches checked (of all): "
          + ", ".join(f"{k} {len(seen[k])}/{total[k]}" for k in TEACHER_KINDS if total[k]))
    print(f"{name} (teacher forward): worst error / bar: " + ", ".join(f"{k} {worst[k]:.3f}" for k in TEACHER_KINDS if total[k])
          + f"; {time.time() - t0:.1f} s")
    del mem, eng, m
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------- injection
def test_external_neck_gradients_are_injected_bit_for_bit():
    t0 = time.time()
    dev = torch.device("cuda:0")
    m = bwd.seeded_model("yolov6m", dev).train()
    eng = m.train_engine()
    eng.external_feat_grads = True
    N, H, W = 2, 96, 160                    # non-square: the NCHW -> NHWC transpose of each level
    with torch.no_grad():
        eng.forward(torch.rand(N, 3, H, W, device=dev))
    gen = torch.Generator(device="cuda").manual_seed(20261020)
    for gb in eng.gbufs:
        gb.fill_(SENT)
    grads = [torch.randn(N, t.c, H >> eng.g.bufs[t.buf].level, W >> eng.g.bufs[t.buf].level, generator=gen, device=dev) * 3
             for t in eng.g.feat]
    eng._feat_grads = list(grads)
    eng.backward(None, None, first=0, last=0)
    torch.cuda.synchronize()
    assert eng._feat_grads is None
    zeroed = {gb.data_ptr() for gb in eng.zero_gbufs}
    expect = {}
    for i, gb in enumerate(eng.gbufs):
        expect[i] = torch.zeros_like(gb) if gb.data_ptr() in zeroed else torch.full_like(gb, SENT)
    for t, gr in zip(eng.g.feat, grads):
        expect[t.buf][..., t.c_off:t.c_off + t.c] = gr.permute(0, 2, 3, 1).to(BF16)
    for i, gb in enumerate(eng.gbufs):
        assert bwd.bits_equal(gb, expect[i]), f"gradient buffer {i}: not the injected gradient / the cleared or untouched rest"
    print(f"\ninjection: {len(grads)} neck slices bit-exact, {len(zeroed)} cleared buffers; {time.time() - t0:.1f} s")
    del eng, m
    torch.cuda.empty_cache()
