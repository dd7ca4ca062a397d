"""CPU checks of the yv6_kl_rows comparison of tests/test_gpu_distill_launches.py, on stand-in tensors: a torch restatement of
the kernel (float64 rows, the fp32 add of each gradient term onto its prior, one accumulation of eff x the row sums) passes
the comparison, and each seeded mistake fails it -- a row the grid-stride loop lost, a mask shifted by one anchor, a
gradient without its 1/T factor (at T = 20: at T = 1 the mistake is invisible) and one stray write into an inactive row."""
import types

import pytest
import torch

import test_gpu_distill_launches as dl

SMS = 132          # the H100 SXM's SMs: the grid the comparison's bars assume


def stand_in(c, e, g0, acc0, skip_row=None, mask=None, inv_t=True):
    """What the kernel leaves: (acc, g).  `skip_row`: a row that is never visited; `mask`: the row mask used instead of the
    case's; `inv_t=False`: the gradient without the factor 1/T."""
    active = e.active.clone()
    if mask is not None:
        active = mask.reshape(-1).repeat_interleave(c.rpm)[:c.rows] != 0
    if skip_row is not None:
        active[skip_row] = False
    term = e.term if inv_t else e.term / c.iT
    g = g0.clone()
    g[active] = g0[active] + term[active].float()
    acc = acc0 + e.eff * float(e.kl[active].sum())
    return torch.tensor(acc, dtype=torch.float64), g


def passes(c, e, acc0, acc, g0, g):
    try:
        dl.assert_untouched(c, e, g0, g, c.name)
    except AssertionError:
        return False
    return dl.kl_value_ratio(c, e, acc0, acc)[0] <= 1.0 and dl.kl_grad_ratio(c, e, g0, g) <= 1.0


def cls_case():
    gen = torch.Generator().manual_seed(1)
    s, t = dl.scores_pair(gen, 256, dl.NC, torch.device("cpu"))
    return dl.kl_case("class T=20", s, t, dl.T_DISTILL, dl.T_DISTILL ** 2)


def dfl_case():
    gen = torch.Generator().manual_seed(2)
    B, A = 2, 96
    fg = dl.fg_mask(gen, B, A, torch.device("cpu"), frac=0.2)
    s, t = dl.dfl_pair(gen, B * A * 4, torch.device("cpu"))
    return dl.kl_case("dfl", s, t, dl.T_DISTILL, dl.T_DISTILL ** 2, mask=fg, rpm=4, num_pos=int(fg.sum()), tss=5.0)


def setup(c):
    e = dl.kl_expected(c, SMS)
    gen = torch.Generator().manual_seed(3)
    mag = float(e.term[e.active].abs().mean())
    g0 = torch.randn(c.rows, c.C, generator=gen) * mag
    acc0 = float(torch.randn(1, generator=gen, dtype=torch.float64))
    return e, g0, acc0


@pytest.mark.parametrize("make", [cls_case, dfl_case])
def test_kl_comparison_passes_the_restated_kernel(make):
    c = make()
    e, g0, acc0 = setup(c)
    acc, g = stand_in(c, e, g0, acc0)
    assert passes(c, e, acc0, acc, g0, g)
    assert dl.kl_value_ratio(c, e, acc0, acc)[1] < 1e-3       # the summed value bar, against the smallest row's term


@pytest.mark.parametrize("make", [cls_case, dfl_case])
def test_kl_comparison_catches_a_dropped_row(make):
    """A row the grid-stride loop never visits: the value alone is off (the summed bar is far below one row's term), and so
    is every element of the row's gradient."""
    c = make()
    e, g0, acc0 = setup(c)
    r = int(e.active.nonzero()[len(e.active.nonzero()) // 2])
    acc, g = stand_in(c, e, g0, acc0, skip_row=r)
    assert dl.kl_value_ratio(c, e, acc0, acc)[0] > 1.0
    assert dl.kl_grad_ratio(c, e, g0, g) > 1.0
    assert not passes(c, e, acc0, acc, g0, g)


def test_kl_comparison_catches_a_mask_shifted_by_one_anchor():
    c = dfl_case()
    e, g0, acc0 = setup(c)
    shifted = torch.roll(c.mask.reshape(-1), 1).reshape(c.mask.shape)
    assert not torch.equal(shifted, c.mask)
    acc, g = stand_in(c, e, g0, acc0, mask=shifted)
    assert not passes(c, e, acc0, acc, g0, g)
    with pytest.raises(AssertionError, match="inactive rows changed"):
        dl.assert_untouched(c, e, g0, g, c.name)


def test_kl_comparison_catches_a_gradient_without_the_inverse_temperature():
    """At T = 20 the term is 20 times too large; the value is right, the gradient is not."""
    c = cls_case()
    e, g0, acc0 = setup(c)
    acc, g = stand_in(c, e, g0, acc0, inv_t=False)
    assert dl.kl_value_ratio(c, e, acc0, acc)[0] <= 1.0
    assert dl.kl_grad_ratio(c, e, g0, g) > 1.0
    # at T = 1 the same mistake cannot be seen: iT = 1
    one = dl.kl_case("class T=1", c.s, c.t, 1.0, 1.0)
    e1 = dl.kl_expected(one, SMS)
    a1, g1 = stand_in(one, e1, g0, acc0, inv_t=False)
    assert passes(one, e1, acc0, a1, g0, g1)


def test_inactive_row_check_catches_one_stray_write():
    c = dfl_case()
    e, g0, acc0 = setup(c)
    acc, g = stand_in(c, e, g0, acc0)
    dl.assert_untouched(c, e, g0, g, c.name)
    r = int((~e.active).nonzero()[3])
    g[r, 5] = torch.nextafter(g[r, 5], torch.tensor(float("inf")))          # one ulp in one element of a masked row
    with pytest.raises(AssertionError, match="inactive rows changed"):
        dl.assert_untouched(c, e, g0, g, c.name)
    # with eff = 0 (gated) every row is inactive
    gated = types.SimpleNamespace(**dict(vars(c), tss=0.0))
    eg = dl.kl_expected(gated, SMS)
    assert eg.eff == 0.0
    g2 = g0.clone()
    g2[int(e.active.nonzero()[0]), 0] += 1.0
    with pytest.raises(AssertionError, match="inactive rows changed"):
        dl.assert_untouched(gated, eg, g0, g2, "gated")
