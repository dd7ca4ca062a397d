"""The conv and weight-gradient kernels keep their wgmma pipelines asynchronous (reads the SASS, no GPU needed).

Two compiler behaviours silently turn the tensor-core pipeline into one MMA at a time, and neither is an error:
  * a function call anywhere in a kernel that issues wgmma (a __noinline__ helper, printf, assert) makes ptxas serialize
    EVERY wgmma of the kernel (warning C7510): each HGMMA carries `gsb0` and is followed by a wait for it;
  * an MMA under a runtime condition inside a commit group makes ptxas split the group and pad it with a dummy
    `HGMMA.64x8x16.F16 RZ` (warning C7519).
This test disassembles the built library with cuobjdump and checks every conv_igemm_kernel / conv_wgrad_kernel variant.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "yolov6_b200", "libyolov6_b200.so")
KERNELS = ("conv_igemm_kernel", "conv_wgrad_kernel")


def _cuobjdump():
    candidates = [shutil.which("cuobjdump")]
    for env in ("CUDA_HOME", "CUDA_PATH"):
        if os.environ.get(env):
            candidates.append(os.path.join(os.environ[env], "bin", "cuobjdump"))
    candidates.append("/usr/local/cuda/bin/cuobjdump")
    return next((c for c in candidates if c and os.access(c, os.X_OK)), None)


@pytest.fixture(scope="module")
def kernels():
    """{mangled kernel name: [SASS lines]} of the wgmma kernels in the built library."""
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("libyolov6_b200.so not built")
    sass = subprocess.run([tool, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs.setdefault(name, [])
        elif name is not None:
            funcs[name].append(line)
    found = {n: body for n, body in funcs.items() if any(k in n for k in KERNELS)}
    for k in KERNELS:
        assert any(k in n for n in found), f"no {k} in the SASS of {LIB}"
    return found


def _instr(line):
    """The instruction text of a SASS line (without the address and encoding comments)."""
    m = re.match(r"\s*/\*[0-9a-f]+\*/\s*(.*?)\s*;", line)
    return m.group(1) if m else None


def test_no_function_calls(kernels):
    bad = [n for n, body in kernels.items() if any((i := _instr(l)) and re.search(r"\bCALL\b", i) for l in body)]
    assert not bad, f"CALL in wgmma kernels (ptxas serializes all their MMAs): {bad}"


def test_mmas_are_chained(kernels):
    """Serialized kernels mark every HGMMA with gsb0; a chained group has gsb0 on its last MMA only."""
    bad = []
    for n, body in kernels.items():
        mmas = [i for i in map(_instr, body) if i and i.startswith("HGMMA")]
        if not mmas or all("gsb0" in i for i in mmas):
            bad.append(n)
    assert not bad, f"no chained HGMMA in: {bad}"


def test_no_dummy_mma(kernels):
    bad = [n for n, body in kernels.items()
           if any((i := _instr(l)) and re.match(r"HGMMA\.64x8x16\.F16\S*\s+RZ\b", i) for l in body)]
    assert not bad, f"dummy HGMMA.64x8x16.F16 RZ (split commit group) in: {bad}"
