"""CPU checks behind the run-to-run identity and the deep-encoder parity tests: which kernels may add with atomics, the
grouped-conv (block-diagonal) weight algebra, and that the GPU parity table covers every layer the engine builds."""
import glob
import os
import re

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "habitat-lab_b200", "csrc")

# Functions allowed to contain atomicAdd / atomicAdd_block / red.global.add, with the reason the result is still the same
# every run.  fp64 statistics: every addend is an fp32 value (or an fp64 sum of fp32 values), i.e. an integer multiple of
# the smallest addend's ulp; fp64 holds such sums exactly, in any order, unless the addends span about 2^25 in magnitude
# (53 - 24 significand bits, less a few bits for the count).  Float gradient sums across blocks are not allowed here:
# they write per-block partials that reduce_partials adds in a fixed order.
ATOMICS_ALLOWED = {
    "conv_igemm_kernel": "fp64 GroupNorm sum / sum of squares of fp32 accumulator partials (exact, see above)",
    "halo_gn_stats_chunk": "fp64 GroupNorm statistics of fp32 partials (exact, see above)",
    "s2_gn_stats_chunk": "fp64 GroupNorm statistics of fp32 partials (exact, see above)",
    "prep_stats_kernel": "fp64 RunningMeanAndVar sums of fp32 pooled pixels (exact, see above)",
    "prep_generic_kernel": "fp64 RunningMeanAndVar sums of fp32 pooled pixels (exact, see above)",
    "gae_serial_kernel": "fp64 advantage sum / count (exact) and sum of squares (last fp64 bit only; consumed in fp32)",
    "gae_warp_kernel": "fp64 advantage sum / count (exact) and sum of squares (last fp64 bit only; consumed in fp32)",
    "grid_barrier": "integer arrival counter of the persistent recurrence's grid barrier",
    "tg_epilogue": "integer split-K tickets: the last CTA of a tile sums the partials in split order",
    "gn_bwd_reduce_kernel": "test-only: the two-pass GroupNorm backward the fused gn_bwd is checked against",
    "lstm_step_bwd_matmul_kernel": "test-only: the per-step LSTM backward the sequence kernels are checked against",
}

_DEF = re.compile(r"(?:__global__|__device__)[^;{}]*\{")
_NAME = re.compile(r"\b(\w+)\s*\(")
_ATOMIC = re.compile(r"atomicAdd_block|atomicAdd\s*\(|red\.global\.add")


def atomic_sites():
    """(file, line, enclosing __global__ / __device__ function) of every atomic add in the CUDA sources"""
    sites = []
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh"))):
        src = open(path).read()
        defs = []
        for m in _DEF.finditer(src):
            names = [n for n in _NAME.findall(m.group(0)) if n != "__launch_bounds__"]
            defs.append((m.start(), names[0] if names else "?"))
        for m in _ATOMIC.finditer(src):
            enclosing = [n for start, n in defs if start < m.start()]
            sites.append((os.path.basename(path), src.count("\n", 0, m.start()) + 1,
                          enclosing[-1] if enclosing else None))
    return sites


def test_scanner_finds_the_known_sites():
    fns = {fn for _, _, fn in atomic_sites()}
    assert {"conv_igemm_kernel", "tg_epilogue", "prep_generic_kernel"} <= fns


def test_float_atomics_only_where_allowed():
    bad = [f"{f}:{line} in {fn}" for f, line, fn in atomic_sites() if fn not in ATOMICS_ALLOWED]
    assert not bad, "atomic adds outside the allow-list (sum per-block partials with reduce_partials): " + ", ".join(bad)


def test_allow_list_has_no_stale_entries():
    fns = {fn for _, _, fn in atomic_sites()}
    assert not set(ATOMICS_ALLOWED) - fns
    for reason in ATOMICS_ALLOWED.values():
        assert reason and "\n" not in reason


def test_test_only_kernels_stay_off_the_product_path():
    """the allow-listed float-atomic kernels are reached through ops.gn_bwd_reduce / ops.lstm_step_bwd only"""
    pkg = os.path.join(ROOT, "habitat-lab_b200")
    for py in glob.glob(os.path.join(pkg, "**", "*.py"), recursive=True):
        if os.path.basename(py) == "ops.py":
            continue
        src = open(py).read()
        assert "gn_bwd_reduce(" not in src and "lstm_step_bwd(" not in src, py


# ---------------------------------------------------------------------------------------------
# block-diagonal algebra of the grouped (ResNeXt) convolutions
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,stride,hw", [(64, 1, 8), (128, 2, 8), (256, 2, 6), (512, 2, 4)])
def test_block_diagonal_weight_matches_grouped_conv(C, stride, hw):
    from habitat_lab_b200.rl.resnet_policy import _Conv

    g = 16
    torch.manual_seed(C)
    conv = nn.Conv2d(C, C, 3, stride, 1, groups=g, bias=False).double()
    c = _Conv(conv, nn.GroupNorm(16, C), (hw, hw))
    c._wd = torch.zeros(C, C, 3, 3, dtype=torch.float64)
    c._gd = torch.empty_like(c._wd)
    x = torch.randn(3, C, hw, hw, dtype=torch.float64, requires_grad=True)
    w = c.dense_weight()
    y_ref = F.conv2d(x, conv.weight, stride=stride, padding=1, groups=g)
    torch.testing.assert_close(F.conv2d(x, w, stride=stride, padding=1), y_ref, rtol=1e-12, atol=1e-12)
    # off-diagonal blocks are zero
    mask = torch.block_diag(*[torch.ones(C // g, C // g, dtype=torch.bool)] * g)
    assert (w[~mask] == 0).all()
    dy = torch.randn_like(y_ref)
    dw_ref = torch.autograd.grad(y_ref, conv.weight, dy)[0]
    wd = w.clone().requires_grad_(True)
    c._gd.copy_(torch.autograd.grad(F.conv2d(x, wd, stride=stride, padding=1), wd, dy)[0])
    conv.weight.grad = torch.zeros_like(conv.weight)
    c.store_grad()
    torch.testing.assert_close(conv.weight.grad, dw_ref, rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------------------------------------
# the GPU parity table covers every layer the engine builds
# ---------------------------------------------------------------------------------------------
def _family(eng, c):
    if c is eng.stem:
        return "stem"
    if c.s2_pair is not None or c.s2_main is not None:
        return "s2_pair"
    if c.halo:
        return "halo"
    return "gather+halo_wgrad" if c.halo_w else "gather"


def _engine_layers(config):
    import habitat_lab_b200 as hb
    from habitat_lab_b200 import synthetic as syn
    from habitat_lab_b200.rl.resnet_policy import EncoderEngine, ResNetEncoder

    spaces, backbone = {2: (syn.pointnav_spaces(256, 256), "resnet18"),
                        3: (syn.objectnav_spaces(256, 256, 6, 21), "resnet50"),
                        4: (syn.imagenav_spaces(256, 256, 4), "resneXt50")}[config]
    pol = hb.PointNavResNetPolicy(*spaces, hidden_size=512, num_recurrent_layers=1, rnn_type="GRU",
                                  resnet_baseplanes=32, backbone=backbone, normalize_visual_inputs=True)
    rows = set()
    for enc in [m for m in pol.modules() if isinstance(m, ResNetEncoder)]:
        eng = EncoderEngine(enc, allow_s2d=False)   # the generic prep's routing (the stem as a gather conv)
        for c in eng.convs:
            rows.add((c.ci_real, c.ci, c.co, c.k, c.stride, c.pad, c.in_hw[0], c.conv_groups, c.groups,
                      _family(eng, c)))
    return rows


@pytest.mark.parametrize("config", [2, 3, 4])
def test_parity_table_covers_the_engine(config):
    from test_gpu_deep_encoders import LAYER_TABLE

    rows = _engine_layers(config)
    if config == 2:   # the fused stride-2 block entry has its own GPU test (test_conv_s2_block_entry)
        rows = {r for r in rows if r[-1] != "s2_pair"}
    missing = rows - set(LAYER_TABLE)
    assert not missing, f"config #{config} builds layers the GPU parity table does not test: {sorted(missing)}"
