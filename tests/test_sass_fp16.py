"""The fp16 conv kernels are the bf16 kernels' pipeline on fp16 operands (reads the SASS, no GPU needed).

conv_f16_igemm_kernel<BN, MODE, CP> shares its body with conv_igemm_kernel (a force-inlined template on the operand dtype), so
it must keep what tests/test_sass_wgmma.py and tests/test_sass_pingpong.py check there: chained HGMMAs without a CALL or a
split-group dummy MMA, no spilled accumulators, the setmaxnreg register split.  Every HGMMA in it is an fp16 one (SASS writes
HGMMA.<shape>.F32 for f16 x f16 -> f32 and HGMMA.<shape>.F32.BF16 for bf16).  The fp16 SPPF kernel spills nothing, the fp16
stems no more than their bf16 twins.
"""
import os
import re
import subprocess

import pytest

from test_sass_wgmma import LIB, _cuobjdump, _instr


@pytest.fixture(scope="module")
def sass():
    """{mangled kernel name: [SASS lines]} of the whole built library."""
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("libyolov6_b200.so not built")
    out = subprocess.run([tool, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs.setdefault(name, [])
        elif name is not None:
            funcs[name].append(line)
    return funcs


def _ops(body):
    return [i for i in map(_instr, body) if i]


def _f16_conv(sass):
    found = {n: body for n, body in sass.items() if "conv_f16_igemm_kernel" in n}
    assert len(found) == 40, f"expected 40 conv_f16_igemm_kernel variants (4 BN x 5 modes x CTA pair or not), found {len(found)}"
    return found


def test_every_hgmma_of_the_fp16_convs_is_fp16(sass):
    bad = {}
    for n, body in _f16_conv(sass).items():
        mmas = [i for i in _ops(body) if i.startswith("HGMMA")]
        wrong = sorted({i.split()[0] for i in mmas if not re.match(r"HGMMA\.64x(32|64|96|128)x16\.F32(\s|$)", i)})
        if not mmas or wrong:
            bad[n] = wrong or "no HGMMA"
    assert not bad, f"HGMMA other than f16 x f16 -> f32 in: {bad}"


def test_fp16_convs_keep_the_mma_pipeline_async(sass):
    calls, serial, dummy = [], [], []
    for n, body in _f16_conv(sass).items():
        ops = _ops(body)
        mmas = [i for i in ops if i.startswith("HGMMA")]
        if any(re.search(r"\bCALL\b", i) for i in ops):
            calls.append(n)
        if all("gsb0" in i for i in mmas):
            serial.append(n)
        if any(re.match(r"HGMMA\.64x8x16\.F16\S*\s+RZ\b", i) for i in ops):
            dummy.append(n)
    assert not calls, f"CALL in: {calls}"
    assert not serial, f"no chained HGMMA in: {serial}"
    assert not dummy, f"dummy HGMMA.64x8x16.F16 RZ (split commit group) in: {dummy}"


def test_fp16_convs_keep_the_register_split_and_spill_nothing(sass):
    spills, split = [], []
    for n, body in _f16_conv(sass).items():
        ops = _ops(body)
        if any(re.match(r"(LDL|STL)\b", i) for i in ops):
            spills.append(n)
        reg = [i for i in ops if i.startswith("USETMAXREG")]
        if not any(".DEALLOC" in i for i in reg) or not any(".TRY_ALLOC" in i for i in reg):
            split.append(n)
    assert not spills, f"local-memory traffic in: {spills}"
    assert not split, f"no setmaxnreg register split (USETMAXREG) in: {split}"


def test_fp16_bn64_halo_convs_issue_m64n128_only(sass):
    """As their bf16 twins (tests/test_sass_conv_swap.py): the BN = 64 halo tiles are computed transposed."""
    found = {n: body for n, body in sass.items() if re.search(r"conv_f16_igemm_kernelILi64ELi[1-4]ELb[01]E", n)}
    assert len(found) == 8
    bad = {n: s for n, body in found.items() if (s := {i.split()[0] for i in _ops(body) if i.startswith("HGMMA")}) != {"HGMMA.64x128x16.F32"}}
    assert not bad, bad


def _spills(body):
    return sum(1 for i in _ops(body) if re.match(r"(LDL|STL)\b", i))


def test_fp16_stem_and_sppf_kernels_spill_no_more_than_their_bf16_twins(sass):
    """The fp16 SPPF kernel spills nothing.  The fp16 stems get the register allocation of their bf16 twins (the same body):
    no more local-memory traffic than those (the 48- and 64-channel stems under __launch_bounds__(256, 2) spill in both)."""
    twins = {"stem_mma_f16_kernel": ("stem_mma_kernel", 4), "stem_mma_async_f16_kernel": ("stem_mma_async_kernel", 24),
             "sppf_pool_f16_kernel": ("sppf_pool_bf16_kernel", 1)}
    for key, (twin, count) in twins.items():
        found = {n: body for n, body in sass.items() if key in n}
        assert len(found) == count, f"expected {count} {key} instances, found {sorted(found)}"
        for n, body in found.items():
            tn = n.replace(key, twin).replace(str(len(key)) + twin, str(len(twin)) + twin)
            assert tn in sass, (n, tn)
            assert _spills(body) <= _spills(sass[tn]), f"{n}: {_spills(body)} local-memory instructions, its bf16 twin {_spills(sass[tn])}"
            if key.startswith("sppf"):
                assert _spills(body) == 0, n
            else:                         # fp16 mma.sync: HMMA.16816.F32 (bf16 would be HMMA.16816.F32.BF16)
                assert any(re.match(r"HMMA\.16816\.F32(\s|$)", i) for i in _ops(body)), n
