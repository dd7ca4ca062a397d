"""The 64-output-channel halo convs compute their tile transposed (reads the SASS, no GPU needed).

A BN = 64 halo tile is D[64 channels x 128 pixels] = weights (A) x input box (B): one wgmma.m64n128k16 per k16 step instead of
two m64n64k16 over pixel rows 0-63 and 64-127 (mma_kblock_t in yolov6_b200/csrc/yv6_conv_igemm.cu).  Its bf16 TMA-store
epilogue writes the (channel x pixel) fragments pixel-major with stmatrix .trans.  This holds for every BN = 64 halo variant:
stride 1 and the stride-2 column-pair view, streamed and resident weights, single CTAs and CTA pairs.
"""
import re

from test_sass_wgmma import _instr, kernels  # noqa: F401  (kernels is a fixture)


def _bn64_halo(kernels):  # noqa: F811
    found = {n: body for n, body in kernels.items() if re.search(r"conv_igemm_kernelILi64ELi[1-4]ELb[01]E", n)}
    assert len(found) == 8, f"expected 8 BN = 64 halo variants (MODE 1-4 x CTA pair or not), found {sorted(found)}"
    return found


def _mma_shapes(body):
    return {m.group(1) for i in map(_instr, body) if i and (m := re.match(r"HGMMA\.(\d+x\d+x\d+)", i))}


def test_bn64_halo_issues_m64n128_only(kernels):  # noqa: F811
    bad = {n: sorted(s) for n, body in _bn64_halo(kernels).items() if (s := _mma_shapes(body)) != {"64x128x16"}}
    assert not bad, f"BN = 64 halo variants not issuing HGMMA.64x128x16 alone: {bad}"


def test_bn64_halo_stages_bf16_with_stmatrix(kernels):  # noqa: F811
    bad = [n for n, body in _bn64_halo(kernels).items() if not any((i := _instr(l)) and i.startswith("STSM") for l in body)]
    assert not bad, f"no stmatrix (STSM) in the transposed epilogue of: {bad}"
