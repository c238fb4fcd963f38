"""The route table of ops.ResnetBlockFn, pinned without a GPU: the harness of tests/test_gpu_resnetblock.py (route
assertions from the ctx attributes and the C-ABI call counts, the dx shadow, determinism, every intermediate and gradient
against fp64) runs above the numpy emulation of the C-ABI (test_host_logic_vq_cpu.VqEmu) at the smallest shape of each
route the emulation covers. The fused route's GroupNorm table prologue has no emulation; it is pinned on the GPU only."""
import collections

import pytest
import torch

import test_gpu_resnetblock as R
from test_host_logic_vq_cpu import vq_emu  # noqa: F401  (fixture)

# launches of the entries that run on the tensor cores, counted the way mas_tc_launch_count counts them
TC_ENTRIES = {"mas_conv3x3_fprop_tc16h", "mas_conv3x3_fprop_tc16", "mas_conv3x3_wgrad_tc16", "mas_gemm_rows_packed"}


@pytest.fixture
def emu_state(vq_emu, state, monkeypatch):  # noqa: F811
    from mas_b200 import _lib as L, ops
    mark = []
    monkeypatch.setattr(ops, "_tc_on", lambda: ops.get_impl() != L.IMPL_SIMT)
    monkeypatch.setattr(L, "tc_launch_count", lambda: sum(n in TC_ENTRIES for n in vq_emu.names))
    monkeypatch.setattr(L, "profile_start", lambda: mark.append(len(vq_emu.names)))
    monkeypatch.setattr(L, "profile_report", lambda tag=None: {k: (c, 0.0) for k, c in
                                                                 collections.Counter(vq_emu.names[mark.pop():]).items()})
    monkeypatch.setattr(torch.cuda, "synchronize", lambda: None)
    # torch's CPU convolutions have no TF32 mode: the yardstick of the fp16 / TF32 stages is plain fp32 here, ~2^13 times more
    # accurate than the emulated fp16 operands; those checks only catch gross errors on the CPU (the GPU test holds them to
    # the real TF32 yardstick)
    monkeypatch.setattr(R, "FACTOR_TF32", 1e4)
    return state


state = R.state

CPU_CASES = [((2, 128, 128, 16, 8), "shadow"), ((2, 128, 256, 16, 8), "shadow"), ((2, 64, 64, 16, 16), "unfused"),
             ((2, 128, 128, 8, 8), "unfused"), ((2, 128, 128, 16, 8), "simt")]


@pytest.mark.parametrize("shape,route", CPU_CASES, ids=R._ids(CPU_CASES))
def test_resnetblock_route_table_emulated(shape, route, emu_state):
    emu_state(route)
    x, prm, g = R._inputs(shape, seed=sum(shape), dev="cpu")
    R._verify(f"emu-{route}-{shape}", shape, route, x, prm, g)


@pytest.mark.parametrize("cond", ["grad", "outlier", "offset"])
def test_resnetblock_conditions_emulated(cond, emu_state):
    shape = (2, 128, 128, 16, 8)
    emu_state("shadow")
    x, prm, g = R.CONDITIONS[cond](*R._inputs(shape, seed=7 * sum(shape), dev="cpu"))
    R._verify(f"emu-shadow-{cond}-{shape}", shape, "shadow", x, prm, g, offset=cond == "offset")
