"""Each Hopper primitive of the CUDA sources (inline PTX of the asynchronous copies, the launch with attributes, the
function-attribute opt-in) is written in one place: common.cuh / wgmma.cuh for the device wrappers, common.cuh for
the launch helper, engine.cu for kernel_opt_in.  A second copy would have to be kept in step by hand."""
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mlx_vlm_b200", "csrc")

# text -> (file that owns it, number of occurrences there)
OWNERS = {
    "mbarrier.try_wait": ("common.cuh", 1),
    "mbarrier.init": ("common.cuh", 1),
    "cp.async.bulk.shared": ("common.cuh", 1),
    "cp.async.bulk.tensor": ("wgmma.cuh", 2),  # tma_2d and tma_3d
    "griddepcontrol.wait": ("common.cuh", 1),
    "createpolicy": ("common.cuh", 1),
    "fence.proxy.async": ("common.cuh", 1),
    "__cvta_generic_to_shared": ("common.cuh", 1),
    "cudaLaunchKernelEx": ("common.cuh", 1),
    "cudaLaunchConfig_t": ("common.cuh", 1),
    "cudaFuncSetAttribute": ("engine.cu", 1),
}


def _code(path):
    """the file without its comments (the PTX strings of asm statements stay)"""
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return re.sub(r"//[^\n]*", "", src)


def _sources():
    names = sorted(n for n in os.listdir(CSRC) if n.endswith((".cu", ".cuh")))
    assert "common.cuh" in names and "wgmma.cuh" in names and "engine.cu" in names
    return {n: _code(os.path.join(CSRC, n)) for n in names}


@pytest.mark.parametrize("text", sorted(OWNERS))
def test_primitive_is_written_once(text):
    found = {n: src.count(text) for n, src in _sources().items() if text in src}
    owner, count = OWNERS[text]
    assert found == {owner: count}, f"{text!r} appears in {found}, expected only in {owner} ({count}x)"
