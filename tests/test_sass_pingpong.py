"""The conv kernel's ping-pong register split holds (reads the SASS, no GPU needed).

Each consumer warpgroup keeps the fp32 accumulators of a whole 128 x BN tile in registers (128 per thread at BN = 128).
That only fits because the producer warpgroup gives registers back and the consumers take them (setmaxnreg, SASS
USETMAXREG).  If ptxas cannot fit a variant, it spills the accumulators to local memory (LDL / STL) without any error.
"""
import re

from test_sass_wgmma import _instr, kernels  # noqa: F401  (kernels is a fixture)


def _conv(kernels):
    found = {n: body for n, body in kernels.items() if "conv_igemm_kernel" in n}
    assert len(found) == 40, f"expected 40 conv_igemm_kernel variants (4 BN x 5 modes x CTA pair or not), found {len(found)}"
    return found


def test_conv_no_local_memory(kernels):  # noqa: F811
    bad = [n for n, body in _conv(kernels).items() if any((i := _instr(l)) and re.match(r"(LDL|STL)\b", i) for l in body)]
    assert not bad, f"local-memory traffic (spilled accumulators) in: {bad}"


def test_conv_register_reallocation(kernels):  # noqa: F811
    bad = []
    for n, body in _conv(kernels).items():
        ops = [i for i in map(_instr, body) if i and i.startswith("USETMAXREG")]
        if not any(".DEALLOC" in i for i in ops) or not any(".TRY_ALLOC" in i for i in ops):
            bad.append(n)
    assert not bad, f"no setmaxnreg register split (USETMAXREG) in: {bad}"
