"""GroupNorm, max-pool and observation-prep kernels (csrc/elementwise.cu) against the float64 reference in
tests/groupnorm_reference.py, at config #2's shapes (ResNet18, RGB-D 256x256: the learner's 4096-frame minibatch and
the actor's 64 frames) and at shapes that force every other dispatch path (tests/test_groupnorm_reference_cpu.py
restates the dispatch rules and checks each case reaches the path named here).

Every comparison is per element against the reference's derived bar (see groupnorm_reference.py), reported as the
worst error / bar; each bar is shown tight by perturbed references that must miss it by at least 10x.  Data patterns:
centred y, y offset so |mean| / std = 3 and 30 per group, one near-constant group per frame (variance below eps), y
quantised to a few fp16 levels (exact ties in pool windows); gamma always has mixed signs and exact zeros, beta both
signs.  The references are evaluated in frame chunks so a 4096-frame case stays within a few GB.
"""
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

import groupnorm_reference as R

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

DEV = "cuda"
FR = 128        # frames per comparison chunk
FR_POOL = 16    # the stem's frames are 8x larger, and the pool reference stacks 9 taps


def LAST_CHUNK(B):
    """frames in the last chunk reduce_partials sums (kReduceChunks = 32 chunks of ceil(B / 32) frames)"""
    return -(-B // 32)

# config #2 layers: (C, H, W, G)
LAYERS = {"layer1": (32, 32, 32, 16), "layer2": (64, 16, 16, 16), "layer3": (128, 8, 8, 16),
          "layer4": (256, 4, 4, 16), "compression": (128, 4, 4, 1)}
# other gn_bwd paths: cluster of 8, ragged last CTA, the fused kernel for C >= 512 and for slices over 200 KB
EXTRA = {"cs8": (32, 64, 64, 16), "ragged": (32, 31, 17, 16), "c512": (512, 8, 8, 32), "c2048": (2048, 4, 4, 32),
         "big_slice": (32, 96, 96, 16)}
PATTERNS = ("centred", "offset3", "offset30", "flat_group", "quantised")

GN_CASES = ([(n, 4096, p) for n in LAYERS for p in PATTERNS] + [(n, 64, "centred") for n in LAYERS]
            + [("cs8", 256, p) for p in ("centred", "offset30")] + [("ragged", 64, p) for p in ("centred", "offset30")]
            + [("c512", 64, p) for p in ("centred", "offset30")] + [("c2048", 64, "offset30")]
            + [("big_slice", 16, p) for p in ("centred", "offset30")])


@pytest.fixture(autouse=True)
def _peak_memory():
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    print(f"\n  peak reserved {torch.cuda.max_memory_reserved() / 2 ** 30:.2f} GB")
    torch.cuda.empty_cache()


def make_y(B, hw, C, G, pattern, gen):
    """fp16 [B, hw, C] in the given data pattern (drawn in frame chunks)"""
    return torch.cat([_make_y(min(256, B - b0), hw, C, G, pattern, gen) for b0 in range(0, B, 256)])


def _make_y(B, hw, C, G, pattern, gen):
    y = torch.randn(B, hw, C, device=DEV, generator=gen)
    if pattern == "centred":
        y *= 1.5
    elif pattern in ("offset3", "offset30"):
        k = 3.0 if pattern == "offset3" else 30.0
        s = torch.rand(B, 1, G, 1, device=DEV, generator=gen) * 1.5 + 0.5
        sign = torch.randint(0, 2, (B, 1, G, 1), device=DEV, generator=gen) * 2.0 - 1.0
        y = ((y.view(B, hw, G, C // G) + k * sign) * s).view(B, hw, C)
    elif pattern == "flat_group":
        y *= 1.5
        cpg = C // G
        y[:, :, :cpg] = 1.0 + (torch.rand(B, hw, cpg, device=DEV, generator=gen) < 0.5) * 2.0 ** -10
    elif pattern == "quantised":
        y = (y * 2).round().clamp(-4, 4) / 2
    return y.half()


def make_affine(C, gen):
    gamma = torch.randn(C, device=DEV, generator=gen) * 0.8
    gamma[::7] = 0.0
    return gamma.contiguous(), (torch.randn(C, device=DEV, generator=gen) * 0.3).contiguous()


class Worst:
    """worst error / bar per output over the chunks, and the guards' margins"""

    def __init__(self, tag):
        self.tag, self.r, self.g = tag, {}, {}

    def add(self, name, got, ref, bar, keep=None):
        d = (got.double() - ref).abs() / bar.clamp_min(1e-300)
        if keep is not None:
            d = d[keep]
        r = d.max().item() if d.numel() else 0.0
        self.r[name] = max(self.r.get(name, 0.0), r)

    def guard(self, name, pert, ref, bar, keep=None):
        d = (pert.double() - ref).abs() / bar.clamp_min(1e-300)
        if keep is not None:
            d = d[keep]
        self.g[name] = d.max().item()

    def finish(self):
        print(f"\n  {self.tag}: error / bar " + ", ".join(f"{k} {v:.3g}" for k, v in self.r.items())
              + "; guards " + ", ".join(f"{k} {v:.3g}x" for k, v in self.g.items()))
        bad = {k: v for k, v in self.r.items() if not v <= 1.0}
        assert not bad, f"{self.tag}: over the bar {bad}"
        weak = {k: v for k, v in self.g.items() if not v >= 10.0}
        assert not weak, f"{self.tag}: perturbed reference misses the bar by less than 10x {weak}"


def f16_bar(ref, e):
    return e * (1 + R.UH) + R.out_bar(ref, "f16")


def bf16_bar(ref, e):
    return e * (1 + R.UB) + R.out_bar(ref, "bf16")


# ---------------------------------------------------------------------------------------------------------------
# gn_apply / gn_residual_relu / gn_bwd
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B,pattern", GN_CASES)
def test_groupnorm(hb, name, B, pattern):
    from habitat_lab_b200 import ops

    C, H, W, G = LAYERS.get(name) or EXTRA[name]
    hw = H * W
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(f"{name} {B} {pattern}".encode()))
    y = make_y(B, hw, C, G, pattern, gen)
    st = R.stats_of(y, G)
    gamma, beta = make_affine(C, gen)
    rd = make_y(B, hw, C, G, "centred", gen)       # downsample branch, pre-norm
    rst = R.stats_of(rd, G)
    rgamma, rbeta = make_affine(C, gen)
    res = make_y(B, hw, C, G, "centred", gen)
    g = make_y(B, hw, C, G, "centred", gen).bfloat16()
    act = make_y(B, hw, C, G, "centred", gen)
    w = Worst(f"{name} B={B} {pattern}")
    fwd = name in LAYERS

    if fwd:
        out, out_b = torch.empty_like(y), torch.empty_like(y, dtype=torch.bfloat16)
        lin = torch.empty_like(y)
        out32 = torch.empty(B, hw, C, device=DEV)
        blk, blk_b, blkd = torch.empty_like(y), torch.empty_like(y, dtype=torch.bfloat16), torch.empty_like(y)
        ops.gn_apply(y, st, gamma, beta, out, B, hw, C, G, relu=True, out_bf16=out_b)
        ops.gn_apply(y, st, gamma, beta, lin, B, hw, C, G, relu=False)
        ops.gn_apply(y, st, gamma, beta, out32, B, hw, C, G, relu=True)
        ops.gn_residual_relu(y, st, gamma, beta, res, blk, B, hw, C, G, out_bf16=blk_b)
        ops.gn_residual_relu(y, st, gamma, beta, rd, blkd, B, hw, C, G, rst, rgamma, rbeta)
        for b0 in range(0, B, FR):
            s = slice(b0, b0 + FR)
            a = (y[s], st[s], gamma, beta, G)
            z, e, _ = R.gn_forward(*a, relu=True)
            w.add("apply_relu_f16", out[s], z, f16_bar(z, e))
            w.add("apply_relu_bf16", out_b[s], z, bf16_bar(z, e))
            w.add("apply_relu_f32", out32[s], z, e)
            zl, el, _ = R.gn_forward(*a, relu=False)
            w.add("apply_f16", lin[s], zl, f16_bar(zl, el))
            zr, er, _ = R.gn_forward(*a, res=res[s])
            w.add("residual_f16", blk[s], zr, f16_bar(zr, er))
            w.add("residual_bf16", blk_b[s], zr, bf16_bar(zr, er))
            zd, ed, _ = R.gn_forward(*a, res=rd[s], res_stats=rst[s], res_gamma=rgamma, res_beta=rbeta)
            w.add("residual_ds_f16", blkd[s], zd, f16_bar(zd, ed))
        # guards on the last frame: every group's statistics taken from its neighbour (G > 1), the downsample residual
        # normalised with the main branch's gamma, eps = 1e-6 on the near-constant group
        L = slice(B - 1, B)
        if G > 1:
            stn = st[L].roll(1, dims=1)
            w.guard("apply:neighbour_stats", R.gn_forward(y[L], stn, gamma, beta, G)[0], z[-1:], f16_bar(z[-1:], e[-1:]))
        w.guard("residual_ds:main_gamma",
                R.gn_forward(y[L], st[L], gamma, beta, G, res=rd[L], res_stats=rst[L], res_gamma=gamma,
                             res_beta=rbeta)[0], zd[-1:], f16_bar(zd[-1:], ed[-1:]))
        if pattern == "flat_group":
            w.guard("apply:eps_1e-6", R.gn_forward(y[L], st[L], gamma, beta, G, eps=1e-6, relu=False)[0], zl[-1:],
                    f16_bar(zl[-1:], el[-1:]))
        del out, out_b, lin, out32, blk, blk_b, blkd

    nband = 0
    for mode in (0, 1, 2):
        dga, dbe = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
        dy, gz = torch.empty_like(g), torch.empty_like(g)
        ops.gn_bwd(g, act, y, st, gamma, beta, dga, dbe, dy, gz, B, hw, C, G, mode)
        dga2, dbe2, dy2 = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.empty_like(g)
        ops.gn_bwd(g, act, y, st, gamma, beta, dga2, dbe2, dy2, None, B, hw, C, G, mode)
        torch.cuda.synchronize()
        assert torch.equal(dy, dy2) and torch.equal(dga, dga2) and torch.equal(dbe, dbe2), "run-to-run identity"
        acc = {k: 0.0 for k in ("dgamma", "dbeta", "e_dgamma", "e_dbeta", "tailA", "tailB")}
        for b0 in range(0, B, FR):
            s = slice(b0, b0 + FR)
            ref = R.gn_backward(g[s], y[s], st[s], gamma, beta, G, mode, act=act[s])
            keep = ~ref["band"]
            nband += int(ref["band"].sum())
            w.add(f"dy_m{mode}", dy[s], ref["dy"], bf16_bar(ref["dy"], ref["e_dy"]), keep)
            assert torch.equal(gz[s][keep], ref["gz"].bfloat16()[keep]), "gz is g times the mask"
            for k in ("dgamma", "dbeta", "e_dgamma", "e_dbeta"):
                acc[k] = acc[k] + ref[k]
            acc["tailA"] = acc["tailA"] + ref["A"][max(0, B - LAST_CHUNK(B) - b0):].sum(0)
            acc["tailB"] = acc["tailB"] + ref["Bx"][max(0, B - LAST_CHUNK(B) - b0):].sum(0)
        w.add(f"dgamma_m{mode}", dga, acc["dgamma"], acc["e_dgamma"])
        w.add(f"dbeta_m{mode}", dbe, acc["dbeta"], acc["e_dbeta"])
        # guards: the last chunk of reduce_partials dropped (skipped where every group of a frame is near-constant:
        # there x_hat's rounding of mu, 300x larger, sets the bar); every group's statistics from its neighbour
        if not (pattern == "flat_group" and G == 1):
            w.guard(f"dgamma_m{mode}:drop_last_chunk", acc["dgamma"] - acc["tailB"], acc["dgamma"], acc["e_dgamma"])
            w.guard(f"dbeta_m{mode}:drop_last_chunk", acc["dbeta"] - acc["tailA"], acc["dbeta"], acc["e_dbeta"])
        L = slice(B - 1, B)
        if G > 1:
            stn = st[L].roll(1, dims=1)
            pert = R.gn_backward(g[L], y[L], stn, gamma, beta, G, mode, act=act[L])["dy"]
            w.guard(f"dy_m{mode}:neighbour_stats", pert, ref["dy"][-1:], bf16_bar(ref["dy"][-1:], ref["e_dy"][-1:]),
                    keep[-1:])
        if pattern == "flat_group":
            pert = R.gn_backward(g[L], y[L], st[L], gamma, beta, G, mode, act=act[L], eps=1e-6)["dy"]
            w.guard(f"dy_m{mode}:eps_1e-6", pert, ref["dy"][-1:], bf16_bar(ref["dy"][-1:], ref["e_dy"][-1:]),
                    keep[-1:])
        del dy, gz, dy2
    n = B * hw * C
    print(f"\n  {name} B={B} {pattern}: {nband} mode-1 band elements of {n}")
    # the band is a few u wide around z = 0 (relative to |mu rstd gamma| and |x rstd gamma|): it holds 1e-7..1e-5
    # of the elements, up to 4e-4 where a whole frame is near-constant (rstd ~ 300)
    assert nband <= max(16, n * 1e-3)
    w.finish()


# ---------------------------------------------------------------------------------------------------------------
# stem: GroupNorm + ReLU + MaxPool2d(3, 2, 1), forward and fused backward
# ---------------------------------------------------------------------------------------------------------------
POOL_CASES = [((64, 64), 4096, p) for p in ("centred", "offset3", "quantised", "flat_group")] + \
             [((64, 64), 64, "centred"), ((33, 47), 64, "centred"), ((33, 47), 64, "quantised")]


@pytest.mark.parametrize("hwp,B,pattern", POOL_CASES)
def test_stem_pool(hb, hwp, B, pattern):
    from habitat_lab_b200 import ops

    H, W = hwp
    C, G = 32, 16
    hw = H * W
    Ho, Wo = R.pool_out_hw(H, W)
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(f"{hwp} {B} {pattern}".encode()))
    y = make_y(B, hw, C, G, pattern, gen)
    st = R.stats_of(y, G)
    gamma, beta = make_affine(C, gen)
    out = torch.empty(B, Ho * Wo, C, device=DEV, dtype=torch.float16)
    out_b = torch.empty_like(out, dtype=torch.bfloat16)
    arg = torch.empty(B, Ho * Wo, C, device=DEV, dtype=torch.uint8)
    ops.gn_relu_maxpool(y, st, gamma, beta, out, arg, B, H, W, C, G, out_bf16=out_b)
    dpool = make_y(B, Ho * Wo, C, G, "centred", gen).bfloat16()
    code = torch.empty_like(arg)
    dead = torch.empty_like(arg, dtype=torch.bool)
    w = Worst(f"pool {H}x{W} B={B} {pattern}")
    n_arg = n_dead_diff = 0
    for b0 in range(0, B, FR_POOL):
        s = slice(b0, b0 + FR_POOL)
        val, bar, cd, amb, dd = R.gn_relu_maxpool(y[s], st[s], gamma, beta, G, H, W)
        w.add("pool_f16", out[s], val, f16_bar(val, bar))
        w.add("pool_bf16", out_b[s], val, bf16_bar(val, bar))
        chk = ~amb
        mism = (arg[s] != cd) & chk
        assert not mism.any(), f"{int(mism.sum())} argmax codes differ from torch's first maximum"
        n_arg += int(chk.sum())
        n_dead_diff += int(((arg[s] != cd) & dd).sum())
        code[s], dead[s] = cd, dd
    # where every tap of a window is below 0 the kernel may record another tap than torch's first one (the slab
    # kernel records the largest x); the ReLU stops the gradient there, so routing through the kernel's codes in
    # those windows gives the same dy bit for bit
    print(f"\n  pool {H}x{W} B={B} {pattern}: {n_arg} argmax codes compared, {n_dead_diff} differ in dead windows")
    fused = R.gn_pool_bwd_plan(H, W, C, G) is not None
    assert fused == ops.gn_relu_maxpool_bwd_supported(H, W, C, G)
    dga, dbe, dy = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.empty(B, hw, C, device=DEV,
                                                                                       dtype=torch.bfloat16)
    if fused:
        ops.gn_relu_maxpool_bwd(dpool, code, y, st, gamma, beta, dga, dbe, dy, B, H, W, C, G)
        dga2, dbe2, dy2 = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.empty_like(dy)
        mixed = torch.where(dead, arg, code)
        ops.gn_relu_maxpool_bwd(dpool, mixed, y, st, gamma, beta, dga2, dbe2, dy2, B, H, W, C, G)
        torch.cuda.synchronize()
        assert torch.equal(dy, dy2) and torch.equal(dga, dga2) and torch.equal(dbe, dbe2)
        del dy2
        gin = None
    else:
        dz = torch.empty_like(dy)
        ops.maxpool_bwd(dpool, code, dz, B, H, W, C)
        for b0 in range(0, B, FR):
            s = slice(b0, b0 + FR)
            r = R.maxpool_route(dpool[s], code[s], H, W)
            assert torch.equal(dz[s], r.bfloat16()), "maxpool_bwd routes and sums the pooled gradient"
        ops.gn_bwd(dz, None, y, st, gamma, beta, dga, dbe, dy, None, B, hw, C, G, 1)
        gin = dz
    acc = {k: 0.0 for k in ("dgamma", "dbeta", "e_dgamma", "e_dbeta", "tailB")}
    for b0 in range(0, B, FR_POOL):
        s = slice(b0, b0 + FR_POOL)
        ref = (R.gn_relu_maxpool_bwd(dpool[s], code[s], y[s], st[s], gamma, beta, G, H, W) if gin is None else
               R.gn_backward(gin[s], y[s], st[s], gamma, beta, G, 1))
        w.add("dy", dy[s], ref["dy"], bf16_bar(ref["dy"], ref["e_dy"]), ~ref["band"])
        for k in ("dgamma", "dbeta", "e_dgamma", "e_dbeta"):
            acc[k] = acc[k] + ref[k]
        acc["tailB"] = acc["tailB"] + ref["Bx"][max(0, B - LAST_CHUNK(B) - b0):].sum(0)
    w.add("dgamma", dga, acc["dgamma"], acc["e_dgamma"])
    w.add("dbeta", dbe, acc["dbeta"], acc["e_dbeta"])
    w.guard("dgamma:drop_last_chunk", acc["dgamma"] - acc["tailB"], acc["dgamma"], acc["e_dgamma"])
    # guard: one live window of the last frame (in a channel with gamma != 0) routed to the wrong tap
    L = slice(B - 1, B)
    live = ((out[L].float() > 0.5) & ~dead[L] & (dpool[L].float().abs() > 0.5) & (gamma != 0)).nonzero()
    p, c = int(live[0, 1]), int(live[0, 2])
    bad = code[L].clone()
    bad[0, p, c] = 4 if int(bad[0, p, c]) != 4 else 0
    pert = R.gn_relu_maxpool_bwd(dpool[L], bad, y[L], st[L], gamma, beta, G, H, W)["dy"]
    last = R.gn_relu_maxpool_bwd(dpool[L], code[L], y[L], st[L], gamma, beta, G, H, W)
    w.guard("dy:wrong_tap", pert, last["dy"], bf16_bar(last["dy"], last["e_dy"]), ~last["band"])
    w.finish()


# ---------------------------------------------------------------------------------------------------------------
# observation prep: 256 x 256 RGB-D from an 8256-row rollout storage
# ---------------------------------------------------------------------------------------------------------------
ROWS, HP, WP = 8256, 256, 256


@pytest.fixture(scope="module")
def storage(hb):
    gen = torch.Generator(device=DEV).manual_seed(17)
    rgb = torch.randint(0, 256, (ROWS, HP, WP, 3), device=DEV, dtype=torch.uint8, generator=gen)
    depth = torch.rand(ROWS, HP, WP, 1, device=DEV, generator=gen)
    yield rgb, depth, gen
    del rgb, depth
    torch.cuda.empty_cache()


def _frame_rows(B, gen):
    """shuffled rows with repeats; the first 32 are past row 8192, whose depth byte offset passes 2^31"""
    rows = torch.randint(0, ROWS, (B,), device=DEV, generator=gen)
    rows[:32] = torch.randint(8193, ROWS, (32,), device=DEV, generator=gen)
    rows[32:40] = rows[:8]
    return rows[torch.randperm(B, device=DEV, generator=gen)].int().contiguous()


@pytest.mark.parametrize("kind,B", [("rgbd", 4096), ("rgb", 256), ("depth", 256)])
def test_prep(hb, storage, kind, B):
    from habitat_lab_b200 import ops

    rgb_s, depth_s, gen = storage
    rgb = rgb_s if kind != "depth" else None
    depth = depth_s if kind != "rgb" else None
    C = {"rgbd": 4, "rgb": 3, "depth": 1}[kind]
    Hq, Wq = HP // 2, WP // 2
    w = Worst(f"prep {kind} B={B}")
    mean = torch.rand(C, device=DEV, generator=gen) * 0.5
    var = torch.rand(C, device=DEV, generator=gen) * 0.1 + 0.005
    count = torch.tensor([7.0], device=DEV)
    rm, rv, rc = mean.clone(), var.clone(), count.clone()
    stats, ss = torch.zeros(17, dtype=torch.float64, device=DEV), torch.zeros(16, device=DEV)
    for step in range(3):      # one update, then two more
        rows = _frame_rows(B, gen)
        pm, pv, pc = rm.double(), rv.double(), float(rc.item())
        ops.prep_stats(rgb, depth, rows, HP, WP, stats)
        ops.prep_finalize(stats, rm, rv, rc, ss, C, Hq * Wq, True)
        sm = torch.zeros(C, dtype=torch.float64, device=DEV)
        sq = torch.zeros_like(sm)
        for b0 in range(0, B, 64):
            x = R.prep_pooled(rgb, depth, rows[b0:b0 + 64]).view(-1, C)
            sm += x.sum(0)
            sq += (x * x).sum(0)
        n_el = B * Hq * Wq
        em, ev, ec = R.running_merge(sm, sq, n_el, B, pm, pv, pc)
        e_mean, e_var = R.running_merge_bars(sm, sq, n_el, pm, pv)
        w.add("run_mean", rm, em, e_mean)
        w.add("run_var", rv, ev, e_var)
        assert rc.item() == ec
        # guard: the merge divided by the old count instead of count + new_count
        w.guard(f"run_mean{step}:old_count", (pc * pm + B * (sm / n_el)) / pc, em, e_mean)
    out = torch.empty(B, Hq, Wq, 8, device=DEV, dtype=torch.float16)
    out_b = torch.empty_like(out, dtype=torch.bfloat16)
    o2d = torch.empty(B, HP // 4, WP // 4, 16, device=DEV, dtype=torch.float16)
    ops.prep_apply(rgb, depth, rows, HP, WP, ss, out, out_bf16=out_b)
    ops.prep_apply(rgb, depth, rows, HP, WP, ss, o2d, s2d=True)
    ident = torch.tensor([1.0] * 8 + [0.0] * 8, device=DEV)
    oid = torch.empty_like(out)
    ops.prep_apply(rgb, depth, rows, HP, WP, ident, oid)
    torch.cuda.synchronize()
    n_cpu_diff = None
    for b0 in range(0, B, 64):
        s = slice(b0, b0 + 64)
        x = R.prep_pooled(rgb, depth, rows[s])
        ref, e = R.prep_normalise(x, rm, rv)
        e = e + 4 * R.U * x.abs() / rv.double().clamp_min(1e-2).sqrt()
        ref8, e8 = R.nhwc8(ref), R.nhwc8(e)
        w.add("out_f16", out[s], ref8, f16_bar(ref8, e8))
        w.add("out_bf16", out_b[s], ref8, bf16_bar(ref8, e8))
        w.add("out_s2d_f16", o2d[s], R.s2d(ref), f16_bar(R.s2d(ref), R.s2d(e)))
        if b0 == 0:   # channel order: rgb swapped for bgr must miss the bar
            perm = [2, 1, 0, 3][:C] if C >= 3 else list(range(C))
            if C >= 3:
                w.guard("out:bgr", R.nhwc8(R.prep_normalise(x[..., perm], rm, rv)[0]), ref8, f16_bar(ref8, e8))
        # identity scale / shift: the pooled fp16 value of ATen's avg_pool2d on the device, bit for bit
        xs = []
        if rgb is not None:
            xs.append(rgb[rows[s].long()].float() * (1.0 / 255.0))
        if depth is not None:
            xs.append(depth[rows[s].long()])
        xf = torch.cat(xs, -1).permute(0, 3, 1, 2)
        pooled = F.avg_pool2d(xf, 2).permute(0, 2, 3, 1).half()
        assert torch.equal(oid[s][..., :C], pooled), "prep's pooled value is torch.cuda's avg_pool2d bit for bit"
        assert (oid[s][..., C:] == 0).all() and (out[s][..., C:] == 0).all()
        if b0 == 0:
            pc_ = F.avg_pool2d(xf[:8].cpu(), 2).permute(0, 2, 3, 1).half()
            n_cpu_diff = int((pc_ != oid[:8, ..., :C].cpu()).sum())
    print(f"\n  prep {kind}: pooled fp16 values differing from the CPU avg_pool2d: {n_cpu_diff} of "
          f"{8 * Hq * Wq * C}")
    w.finish()


# ---------------------------------------------------------------------------------------------------------------
# NaN: the ReLU and the pool maxima propagate NaN as torch.relu / MaxPool2d do
# ---------------------------------------------------------------------------------------------------------------
def _nan_case(B, H, W, C, G, gen):
    y = make_y(B, H * W, C, G, "centred", gen)
    st = R.stats_of(y, G)
    y[0, 5, 3] = float("nan")                 # one element of frame 0
    st[1, 2] = float("nan")                   # frame 1, group 2
    gamma, beta = make_affine(C, gen)
    gamma[3] = 0.7                            # channel 3 of the NaN element has gamma != 0
    return y, st, gamma, beta


def _torch_gn_relu(y, st, gamma, beta, G, H, W):
    """float64 relu(GN(y)) NCHW from the given statistics, NaN propagating (torch semantics)"""
    z = R.gn_forward(y, st, gamma, beta, G, relu=False)[0]
    return F.relu(z.view(y.shape[0], H, W, -1).permute(0, 3, 1, 2))


def test_nan_apply_and_residual(hb):
    from habitat_lab_b200 import ops

    B, H, W, C, G = 3, 8, 8, 64, 16
    gen = torch.Generator(device=DEV).manual_seed(31)
    y, st, gamma, beta = _nan_case(B, H, W, C, G, gen)
    res = make_y(B, H * W, C, G, "centred", gen)
    res[2, 7, 9] = float("nan")
    ref = _torch_gn_relu(y, st, gamma, beta, G, H, W).permute(0, 2, 3, 1).reshape(B, H * W, C)
    expect = ref.isnan()
    assert expect.sum() == 1 + H * W * (C // G)
    for relu in (False, True):          # the relu output is checked below
        out, out_b = torch.empty_like(y), torch.empty_like(y, dtype=torch.bfloat16)
        ops.gn_apply(y, st, gamma, beta, out, B, H * W, C, G, relu=relu, out_bf16=out_b)
        assert torch.equal(out.isnan(), expect) and torch.equal(out_b.isnan(), expect)
    blk = torch.empty_like(y)
    ops.gn_residual_relu(y, st, gamma, beta, res, blk, B, H * W, C, G)
    zr = R.gn_forward(y, st, gamma, beta, G, res=res)[0]
    zr = torch.where((y.double() + res.double()).isnan() | R.gn_forward(y, st, gamma, beta, G, relu=False)[0].isnan(),
                     math.nan, zr)
    assert torch.equal(blk.isnan(), zr.isnan()) and int(blk.isnan().sum()) == 2 + H * W * (C // G)
    # finite elements are unaffected
    keep = ~expect
    assert ((out.double() - ref.nan_to_num()).abs()[keep] <= 2e-3 * (1 + ref.nan_to_num().abs()[keep])).all()


@pytest.mark.parametrize("H,W", [(16, 16), (9, 13)], ids=["slab", "generic"])
def test_nan_pool(hb, H, W):
    from habitat_lab_b200 import ops

    B, C, G = 3, 32, 16
    assert R.gn_pool_fwd_path(C, H, W)[0] == ("slab" if H % 2 == 0 else "generic")
    gen = torch.Generator(device=DEV).manual_seed(32)
    y, st, gamma, beta = _nan_case(B, H, W, C, G, gen)
    y[0, 5 + W, 3] = float("nan")             # a second NaN in the same channel, one row below
    Ho, Wo = R.pool_out_hw(H, W)
    out = torch.empty(B, Ho * Wo, C, device=DEV, dtype=torch.float16)
    out_b = torch.empty_like(out, dtype=torch.bfloat16)
    arg = torch.empty(B, Ho * Wo, C, device=DEV, dtype=torch.uint8)
    ops.gn_relu_maxpool(y, st, gamma, beta, out, arg, B, H, W, C, G, out_bf16=out_b)
    z = _torch_gn_relu(y, st, gamma, beta, G, H, W)
    p, idx = F.max_pool2d(z.cpu(), 3, 2, 1, return_indices=True)      # CPU and CUDA MaxPool2d: the last NaN tap wins
    p = p.permute(0, 2, 3, 1).reshape(B, Ho * Wo, C).to(DEV)
    oy = torch.arange(Ho).view(1, 1, Ho, 1)
    ox = torch.arange(Wo).view(1, 1, 1, Wo)
    code = ((idx // W - (2 * oy - 1)) * 3 + (idx % W - (2 * ox - 1))).permute(0, 2, 3, 1).reshape(B, Ho * Wo, C)
    nan = p.isnan()
    assert nan[0].sum() >= 2 and nan[1].sum() == Ho * Wo * (C // G)
    assert torch.equal(out.isnan(), nan) and torch.equal(out_b.isnan(), nan)
    assert torch.equal(arg[nan].cpu().long(), code.to(DEV)[nan].cpu())


# ---------------------------------------------------------------------------------------------------------------
# GroupNorm statistics from the conv epilogues at 4096 frames
# ---------------------------------------------------------------------------------------------------------------
# name: (kernel, input C, H, W, output N, groups); config #2's convolutions that write GroupNorm statistics
CONV_STATS = {
    "stem_halo_s2d": ("stem", 4, 128, 128, 32, 16),   # 7x7 stride-2 over the 256x256 prep output as 4x4 over s2d
    "layer1_halo": ("halo", 32, 32, 32, 32, 16),
    "layer2_halo": ("halo", 64, 16, 16, 64, 16),
    "layer2_entry_s2": ("s2", 32, 32, 32, 64, 16),    # 3x3 stride-2 + 1x1 stride-2 downsample, both statistics
    "layer3_conv": ("conv", 128, 8, 8, 128, 16),
    "layer4_conv": ("conv", 256, 4, 4, 256, 16),
    "compression_conv": ("conv", 256, 4, 4, 128, 1),
}


def _stats_check(w, name, stats, y_ref_chunks, G):
    """stats [B, G, 2] against float64 sums of the fp32 reference outputs (NCHW chunks), bar 1e-4 * sum|terms| + 1e-6
    as in test_layer_parity; the guard credits the last frame's first pixels (up to 64, half a tile) to the frame
    before it"""
    refs, bars = [], []
    for yr in y_ref_chunks:
        yg = yr.double().reshape(yr.shape[0], G, -1)
        refs.append(torch.stack([yg.sum(-1), (yg * yg).sum(-1)], -1))
        bars.append(1e-4 * torch.stack([yg.abs().sum(-1), (yg * yg).sum(-1)], -1) + 1e-6)
        last = yr[-1].double()
    ref, bar = torch.cat(refs), torch.cat(bars)
    w.add(name, stats, ref, bar)
    N = last.shape[0]
    npx = min(64, last[0].numel() // 2)
    moved = last.reshape(N, -1)[:, :npx].reshape(G, -1)
    mv = torch.stack([moved.sum(-1), (moved * moved).sum(-1)], -1)
    pert = ref[-2:].clone()
    pert[-1] -= mv
    pert[-2] += mv
    w.guard(name + ":tile_to_wrong_frame", pert, ref[-2:], bar[-2:])


@pytest.mark.parametrize("name", list(CONV_STATS))
def test_conv_epilogue_stats(hb, name):
    from habitat_lab_b200 import ops

    kind, C, H, W, N, G = CONV_STATS[name]
    B, FRC = 4096, 128
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(name.encode()))
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    w = Worst(f"conv stats {name} B={B}")
    try:
        x = make_y(B, H * W, C, 1, "centred", gen).view(B, H, W, C)     # fp16 NHWC
        if kind == "stem":
            wt = torch.randn(N, C, 7, 7, device=DEV, generator=gen) / math.sqrt(C * 49)
            img = torch.empty(16 * 16 * N, device=DEV, dtype=torch.float16)
            ops.pack_halo_weight(wt, img, 16, N, 4, 2)
            Ho, Wo = H // 2, W // 2
            xs = x.view(B, Ho, 2, Wo, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, Ho, Wo, 4 * C).contiguous()
            y = torch.empty(B, Ho, Wo, N, device=DEV, dtype=torch.float16)
            st = torch.zeros(B, G, 2, device=DEV, dtype=torch.float64)
            ops.conv_halo(xs, img, y, B, Ho, Wo, 4 * C, N, 4, 0, gn_stats=st, gn_groups=G)
            del xs
            outs = [(st, lambda xc: F.conv2d(xc, wt.half().float(), stride=2, padding=3))]
        elif kind == "halo":
            wt = torch.randn(N, C, 3, 3, device=DEV, generator=gen) / math.sqrt(C * 9)
            img = torch.empty(9 * C * N, dtype=torch.float16, device=DEV)
            ops.pack_halo_weight(wt, img, C, N, 3, 0)
            y = torch.empty(B, H, W, N, device=DEV, dtype=torch.float16)
            st = torch.zeros(B, G, 2, device=DEV, dtype=torch.float64)
            ops.conv_halo(x, img, y, B, H, W, C, N, 3, 0, gn_stats=st, gn_groups=G)
            outs = [(st, lambda xc: F.conv2d(xc, wt.half().float(), padding=1))]
        elif kind == "s2":
            assert ops.conv_s2_supported(C, N, N, H, W)
            wa = torch.randn(N, C, 3, 3, device=DEV, generator=gen) / math.sqrt(9 * C)
            wd = torch.randn(N, C, 1, 1, device=DEV, generator=gen) / math.sqrt(C)
            wcat = torch.zeros(2 * N, C, 3, 3, device=DEV)
            wcat[:N] = wa
            wcat[N:, :, 1, 1] = wd[:, :, 0, 0]
            img = torch.empty(9 * C * 2 * N, device=DEV, dtype=torch.float16)
            ops.pack_halo_weight(wcat, img, C, 2 * N, 3, 0)
            ya = torch.empty(B, H // 2, W // 2, N, device=DEV, dtype=torch.float16)
            yb = torch.empty_like(ya)
            sa = torch.zeros(B, G, 2, device=DEV, dtype=torch.float64)
            sb = torch.zeros_like(sa)
            ops.conv_s2_fwd(x, img, ya, yb, B, H, W, C, N, N, stats_a=sa, groups_a=G, stats_b=sb, groups_b=G)
            outs = [(sa, lambda xc: F.conv2d(xc, wa.half().float(), stride=2, padding=1)),
                    (sb, lambda xc: F.conv2d(xc, wd.half().float(), stride=2))]
        else:
            wt = torch.randn(N, C, 3, 3, device=DEV, generator=gen) / math.sqrt(C * 9)
            s = ops.conv_shape(B, H, W, C, N, 3, 3, 1, 1)
            wp, _ = ops.pack_conv_weight(wt, C, want_t=False)
            y = torch.empty(B, H, W, N, device=DEV, dtype=torch.float16)
            st = torch.zeros(B, G, 2, device=DEV, dtype=torch.float64)
            ops.conv_fwd(x, wp, y, s, st, G)
            outs = [(st, lambda xc: F.conv2d(xc, wt.half().float(), padding=1))]
        torch.cuda.synchronize()
        for j, (st, conv) in enumerate(outs):
            chunks = (conv(x[b0:b0 + FRC].permute(0, 3, 1, 2).float()) for b0 in range(0, B, FRC))
            _stats_check(w, ("stats", "stats_downsample")[j], st, chunks, G)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    w.finish()
