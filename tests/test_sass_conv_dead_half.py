"""The pixel-major conv variants carry a second K loop for tiles whose rows 64-127 lie wholly outside the output (reads the SASS,
no GPU needed).

On a map with Ho % 16 in 1..8 (the 40 x 40 maps of YOLOv6-S/M at 640), the last row of 8 x 16 halo tiles has only its pixel
rows 0-63 inside the output.  Each consumer warpgroup decides once per tile and then runs one of two copies of the K loop,
each with a compile-time MMA count per commit group: the full one issues two m64nBNk16 per k16 step (rows 0-63 into one
accumulator, rows 64-127 into the other), the rows 0-63 one issues the first of them only (mma_kblock<..., LO = true> in
yolov6_b200/csrc/yv6_conv_igemm.cu).  A runtime `if` around the second MMA would make ptxas split the group instead
(test_sass_wgmma.py), and a second copy of the loop must not push the accumulators out of registers (test_sass_pingpong.py).
The transposed BN = 64 halo variants issue one m64n128 over all 128 pixels and have no such loop (test_sass_conv_swap.py).
"""
import re
from collections import Counter

from test_sass_wgmma import _instr, kernels  # noqa: F401  (kernels is a fixture)

HALO_TAPS = {1: 9, 2: 9, 3: 6, 4: 6}     # taps per 64-channel block: 3x3 stride 1, 3x2 on the column-pair view


def _variants(kernels, bn, modes):  # noqa: F811
    pat = re.compile(rf"conv_igemm_kernelILi{bn}ELi([{modes}])ELb([01])E")
    found = {n: (int(m.group(1)), body) for n, body in kernels.items() if (m := pat.search(n))}
    assert len(found) == 2 * len(modes), f"expected {2 * len(modes)} BN = {bn} variants of modes {modes}, found {sorted(found)}"
    return found


def _groups(body):
    """The commit groups of a kernel in program order: the accumulator registers of each HGMMA up to the one carrying gsb0."""
    groups, cur = [], []
    for i in map(_instr, body):
        if i and i.startswith("HGMMA"):
            cur.append(re.match(r"HGMMA\.\S+\s+(R\d+),", i).group(1))
            if "gsb0" in i:
                groups.append(cur)
                cur = []
    return groups


def _check_two_loops(name, groups, full_sizes):
    """full_sizes: {MMAs per group of the full-tile loop: groups of that size}.  The rows 0-63 loop has as many groups of half
    the size, each into a single accumulator that is also the first accumulator of the full groups."""
    sizes = Counter(len(g) for g in groups)
    want = Counter(full_sizes) + Counter({s // 2: c for s, c in full_sizes.items()})
    assert sizes == want, f"{name}: commit groups by size {dict(sizes)}, expected {dict(want)}"
    # the full groups alternate two accumulators (rows 0-63, rows 64-127); a half group uses one of them only
    full = [g for g in groups if len(g) == max(full_sizes) and len(set(g)) == 2]
    assert full, f"{name}: no full-tile group alternating two accumulators"
    lo_acc = {g[0] for g in full}
    halves = [g for g in groups if len(g) == max(full_sizes) // 2 and len(set(g)) == 1 and g[0] in lo_acc]
    assert len(halves) == full_sizes[max(full_sizes)], f"{name}: rows 0-63 groups {halves} do not write the rows 0-63 accumulator"


def test_bn128_halo_has_rows_0_63_loop(kernels):  # noqa: F811
    for n, (mode, body) in _variants(kernels, 128, "1234").items():
        _check_two_loops(n, _groups(body), {8: HALO_TAPS[mode]})      # 2 x 4 k16 steps per tap, 4 in the rows 0-63 loop


def test_bn96_halo_has_rows_0_63_loop(kernels):  # noqa: F811
    for n, (mode, body) in _variants(kernels, 96, "1234").items():
        _check_two_loops(n, _groups(body), {8: HALO_TAPS[mode]})


def test_mode0_has_rows_0_63_loop(kernels):  # noqa: F811
    # 16-, 32- and 64-channel K blocks (1, 2 or 4 k16 steps) in each loop
    for bn in (32, 64, 96, 128):
        for n, (_mode, body) in _variants(kernels, bn, "0").items():
            _check_two_loops(n, _groups(body), {2: 1, 4: 1, 8: 1})


def test_two_loops_keep_the_register_budget(kernels):  # noqa: F811
    """No CALL (which would serialize every MMA), no local memory, and the setmaxnreg split still in place."""
    for bn in (32, 64, 96, 128):
        for n, (_mode, body) in _variants(kernels, bn, "01234").items():
            ins = [i for i in map(_instr, body) if i]
            assert not any(re.search(r"\bCALL\b", i) for i in ins), f"CALL in {n}"
            assert not any(re.match(r"(LDL|STL)\b", i) for i in ins), f"local-memory traffic in {n}"
            assert any(i.startswith("USETMAXREG.DEALLOC") for i in ins), f"no USETMAXREG.DEALLOC in {n}"
            assert any(i.startswith("USETMAXREG.TRY_ALLOC") for i in ins), f"no USETMAXREG.TRY_ALLOC in {n}"
