"""CPU checks of the float64 GroupNorm / max-pool / prep reference that tests/test_gpu_groupnorm.py judges the
elementwise.cu kernels by: the reference equals torch (forward and autograd gradients, every mask mode, the pool's
first-maximum rule), chunked equals unchunked, fp32 evaluations of the kernels' formulas stay within the bars, prep
equals the oracle's RunningMeanAndVar, and every shape of the GPU tests reaches the dispatch path it claims."""
import pytest
import torch
import torch.nn.functional as F

import groupnorm_reference as R
from oracle import torch_oracle as O


def _case(B, C, h, w, seed, offset=0.0, quant=False):
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(B, h * w, C, generator=g, dtype=torch.float64) * 1.5 + offset
    if quant:
        y = (y * 2).round().clamp(-4, 4) / 2
    y = y.half().double()
    gamma = (torch.randn(C, generator=g) * 0.8).float()
    gamma[::7] = 0.0
    beta = (torch.randn(C, generator=g) * 0.3).float()
    return y, gamma, beta, g


def _nchw(t, h, w):
    B, _, C = t.shape
    return t.view(B, h, w, C).permute(0, 3, 1, 2)


def _nhwc(t):
    B, C, h, w = t.shape
    return t.permute(0, 2, 3, 1).reshape(B, h * w, C)


@pytest.mark.parametrize("B,C,h,w,G", [(3, 32, 6, 5, 16), (2, 64, 4, 4, 16), (2, 16, 3, 7, 1)])
def test_forward_is_group_norm(B, C, h, w, G):
    y, gamma, beta, g = _case(B, C, h, w, 1)
    res = torch.randn(B, h * w, C, generator=g, dtype=torch.float64)
    yd = torch.randn(B, h * w, C, generator=g, dtype=torch.float64) * 2 + 1
    gd, bd = torch.randn(C, generator=g).float(), torch.randn(C, generator=g).float()
    st, rst = R.stats_of(y, G), R.stats_of(yd, G)
    tol = dict(rtol=1e-12, atol=1e-12)
    gn = lambda t, ga, be: _nhwc(F.group_norm(_nchw(t, h, w), G, ga.double(), be.double(), eps=1e-5))  # noqa: E731
    torch.testing.assert_close(R.gn_forward(y, st, gamma, beta, G, relu=False)[0], gn(y, gamma, beta), **tol)
    torch.testing.assert_close(R.gn_forward(y, st, gamma, beta, G)[0], gn(y, gamma, beta).relu(), **tol)
    torch.testing.assert_close(R.gn_forward(y, st, gamma, beta, G, res=res)[0], (gn(y, gamma, beta) + res).relu(),
                               **tol)
    torch.testing.assert_close(R.gn_forward(y, st, gamma, beta, G, res=yd, res_stats=rst, res_gamma=gd, res_beta=bd)[0],
                               (gn(y, gamma, beta) + gn(yd, gd, bd)).relu(), **tol)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("B,C,h,w,G", [(3, 32, 6, 5, 16), (2, 16, 4, 4, 1)])
def test_backward_is_autograd(mode, B, C, h, w, G):
    y, gamma, beta, g = _case(B, C, h, w, 2 + mode, offset=0.7)
    dout = torch.randn(B, h * w, C, generator=g, dtype=torch.float64)
    act = torch.randn(B, h * w, C, generator=g, dtype=torch.float64)
    yr = y.clone().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    z = _nhwc(F.group_norm(_nchw(yr, h, w), G, gr, br, eps=1e-5))
    if mode == 1:
        z = z.relu()
    (z * dout * ((act > 0) if mode == 2 else 1)).sum().backward()
    ref = R.gn_backward(dout, y, R.stats_of(y, G), gamma, beta, G, mode, act=act)
    tol = dict(rtol=1e-10, atol=1e-11)
    torch.testing.assert_close(ref["dy"], yr.grad, **tol)
    torch.testing.assert_close(ref["dgamma"], gr.grad, **tol)
    torch.testing.assert_close(ref["dbeta"], br.grad, **tol)


def test_chunked_equals_unchunked(monkeypatch):
    B, C, h, w, G = 7, 32, 6, 6, 16
    y, gamma, beta, g = _case(B, C, h, w, 9)
    dp = torch.randn(B, 9, C, generator=g, dtype=torch.float64)
    st = R.stats_of(y, G)
    whole = (R.gn_forward(y, st, gamma, beta, G), R.gn_relu_maxpool(y, st, gamma, beta, G, h, w),
             R.gn_backward(dp.repeat(1, 4, 1), y, st, gamma, beta, G, 1))
    monkeypatch.setattr(R, "CHUNK", 3)
    parts = (R.gn_forward(y, st, gamma, beta, G), R.gn_relu_maxpool(y, st, gamma, beta, G, h, w),
             R.gn_backward(dp.repeat(1, 4, 1), y, st, gamma, beta, G, 1))
    assert torch.equal(R.stats_of(y, G), st)
    for a, b in zip(whole[0] + whole[1], parts[0] + parts[1]):
        assert torch.equal(a, b)
    for k in ("dy", "gz", "e_dy", "A", "Bx"):
        assert torch.equal(whole[2][k], parts[2][k])
    for k in ("dgamma", "dbeta", "e_dgamma", "e_dbeta"):
        torch.testing.assert_close(whole[2][k], parts[2][k], rtol=1e-14, atol=0)


@pytest.mark.parametrize("h,w", [(8, 6), (7, 5)])
def test_pool_is_max_pool2d_first_maximum(h, w):
    """values, tap codes with ties (quantised y, gamma = 0 channels) and the fused backward against torch on the CPU,
    whose max_pool2d keeps the first of equal taps"""
    B, C, G = 3, 16, 8
    y, gamma, beta, g = _case(B, C, h, w, 4, quant=True)
    st = R.stats_of(y, G)
    val, bar, code, amb, dead = R.gn_relu_maxpool(y, st, gamma, beta, G, h, w)
    yr = y.clone().requires_grad_(True)
    z = F.group_norm(_nchw(yr, h, w), G, gamma.double(), beta.double(), eps=1e-5).relu()
    p, idx = F.max_pool2d(z, 3, 2, 1, return_indices=True)
    Ho, Wo = R.pool_out_hw(h, w)
    torch.testing.assert_close(val, _nhwc(p.detach()), rtol=1e-12, atol=1e-12)
    oy = torch.arange(Ho).view(1, 1, Ho, 1)
    ox = torch.arange(Wo).view(1, 1, 1, Wo)
    tcode = (idx // w - (2 * oy - 1)) * 3 + (idx % w - (2 * ox - 1))
    assert torch.equal(code.long(), _nhwc(tcode))
    ties = (R._taps(R.gn_forward(y, st, gamma, beta, G)[0], h, w, -1.0) == val.view(B, Ho, Wo, C)).sum(0) > 1
    assert ties.sum() > 50  # the quantised data do exercise the tie rule
    assert dead.any() and not (dead & (val != 0)).any()
    dp = torch.randn(B, Ho * Wo, C, generator=g, dtype=torch.float64)
    p.backward(_nchw(dp, Ho, Wo))
    ref = R.gn_relu_maxpool_bwd(dp, code, y, st, gamma, beta, G, h, w)
    torch.testing.assert_close(ref["dy"], yr.grad, rtol=1e-10, atol=1e-11)


def test_fp32_formulas_within_bars():
    """the kernels' two fp32 formulas for z, and a two-pass fp32 backward, stay within the bars at |mean| / std up to
    30 and on a group whose variance is below eps; at least 4x inside the bar"""
    B, C, h, w, G = 4, 32, 9, 7, 16
    for offset in (0.0, 3.0, 30.0):
        y, gamma, beta, g = _case(B, C, h, w, 5, offset=offset)
        y[:, :, :2] = (1.0 + (torch.rand(B, h * w, 2, generator=g) < 0.5) * 2.0 ** -10).half().double()
        st = R.stats_of(y, G)
        z, e, _ = R.gn_forward(y, st, gamma, beta, G, relu=False)
        m = (C // G) * h * w
        mean = (st[..., 0] / m).float().repeat_interleave(C // G, 1)[:, None]
        var = (st[..., 1] / m - (st[..., 0] / m) ** 2).float().clamp_min(0).repeat_interleave(C // G, 1)[:, None]
        rs = torch.rsqrt(var + 1e-5)
        x = y.float()
        z1 = torch.addcmul(beta, (x - mean) * rs, gamma)
        sc = rs * gamma
        z2 = torch.addcmul(beta - mean * sc, x, sc)
        for zz in (z1, z2):
            assert ((zz.double() - z).abs() <= e / 4).all()
        dout = torch.randn(B, h * w, C, generator=g).bfloat16().double()
        ref = R.gn_backward(dout, y, st, gamma, beta, G, 1)
        xh = (x - mean) * rs
        gz = dout.float() * ((xh * gamma + beta) > 0)
        A, Bx = gz.sum(1), (gz * xh).sum(1)
        keep = ~ref["band"]
        assert ((A.double() - ref["A"]).abs() <= ref["e_A"] / 4).all()
        assert ((Bx.double() - ref["Bx"]).abs() <= ref["e_Bx"] / 4).all()
        S1 = (gamma * A).view(B, G, -1).sum(-1).repeat_interleave(C // G, 1)[:, None]
        S2 = (gamma * Bx).view(B, G, -1).sum(-1).repeat_interleave(C // G, 1)[:, None]
        dy = rs * gamma * gz - rs / m * (S1 + xh * S2)
        assert ((dy.double() - ref["dy"]).abs() <= ref["e_dy"] / 4)[keep].all()


def test_prep_is_running_mean_and_var():
    g = torch.Generator().manual_seed(6)
    N, H, W = 9, 16, 24
    rgb = torch.randint(0, 256, (N, H, W, 3), generator=g, dtype=torch.uint8)
    depth = torch.rand(N, H, W, 1, generator=g)
    rows = torch.tensor([4, 0, 8, 4, 2], dtype=torch.int32)
    x = R.prep_pooled(rgb, depth, rows)
    xo = F.avg_pool2d(torch.cat([rgb[rows.long()].permute(0, 3, 1, 2).double() / 255.0,
                                 depth[rows.long()].permute(0, 3, 1, 2).double()], 1), 2)
    torch.testing.assert_close(x, xo.permute(0, 2, 3, 1), rtol=1e-14, atol=1e-15)
    mean, var, count = torch.rand(4, dtype=torch.float64), torch.rand(4, dtype=torch.float64) + 0.01, 7.0
    n_el = x.shape[0] * x.shape[1] * x.shape[2]
    xs = x.reshape(-1, 4)
    m2, v2, c2 = R.running_merge(xs.sum(0), (xs * xs).sum(0), n_el, x.shape[0], mean, var, count)
    om, ov, oc = O.running_mean_var_update(xo, mean.view(1, 4, 1, 1), var.view(1, 4, 1, 1),
                                           torch.tensor(count, dtype=torch.float64))
    torch.testing.assert_close(m2, om.view(-1), rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(v2, ov.view(-1), rtol=1e-12, atol=1e-14)
    assert c2 == oc.item() == count + 5
    out, _ = R.prep_normalise(x, m2, v2)
    torch.testing.assert_close(out, O.running_mean_var_apply(xo, om, ov).permute(0, 2, 3, 1), rtol=1e-12, atol=1e-13)
    s = R.s2d(out)
    assert s.shape == (5, H // 4, W // 4, 16)
    assert torch.equal(s[:, 1, 2, 4 + 2], out[:, 2, 5, 2]) and torch.equal(s[:, 1, 2, 8 + 3], out[:, 3, 4, 3])
    assert torch.equal(R.nhwc8(out)[..., :4], out) and (R.nhwc8(out)[..., 4:] == 0).all()


# ---- dispatch: every case of the GPU tests reaches the path it claims ----------------------------------------
# (C, G, H, W, mask mode) -> gn_bwd path; config #2 at 256 x 256 RGB-D is layer1 32 @ 32x32 ... layer4 256 @ 4x4
GN_BWD_PATHS = [
    ((32, 16, 32, 32, 1), ("cluster", 4)), ((32, 16, 32, 32, 2), ("cluster", 4)),
    ((64, 16, 16, 16, 0), ("cluster", 2)), ((64, 16, 16, 16, 1), ("cluster", 2)), ((64, 16, 16, 16, 2), ("cluster", 2)),
    ((128, 16, 8, 8, 0), ("cluster", 1)), ((128, 16, 8, 8, 1), ("cluster", 1)), ((128, 16, 8, 8, 2), ("cluster", 1)),
    ((256, 16, 4, 4, 0), ("cluster", 1)), ((256, 16, 4, 4, 1), ("cluster", 1)), ((256, 16, 4, 4, 2), ("cluster", 1)),
    ((128, 1, 4, 4, 1), ("cluster", 1)),
    ((32, 16, 64, 64, 1), ("cluster", 8)),       # stem shape through gn_bwd (after maxpool_bwd)
    ((32, 16, 31, 17, 1), ("cluster", 2)),       # ragged last CTA: hw % cs != 0
    ((32, 16, 33, 47, 1), ("cluster", 8)),       # odd stem shape: maxpool_bwd + gn_bwd, ragged
    ((512, 32, 8, 8, 1), ("fused", None)),       # C >= 512 (configs #3 / #4)
    ((2048, 32, 4, 4, 2), ("fused", None)),
    ((32, 16, 96, 96, 2), ("fused", None)),      # slice over 200 KB even at a cluster of 8
]


@pytest.mark.parametrize("shape,path", GN_BWD_PATHS)
def test_gn_bwd_dispatch(shape, path):
    C, G, H, W, mode = shape
    kind, cs, ppc = R.gn_bwd_path(C, G, H * W, mode)
    assert (kind, cs) == path
    if kind == "cluster" and (H, W) == (31, 17):
        assert (H * W) % cs != 0 and ppc * cs > H * W


def test_pool_dispatch():
    assert R.gn_pool_fwd_path(32, 64, 64) == ("slab", 8)       # config #2 stem
    assert R.gn_pool_fwd_path(32, 16, 16) == ("slab", 8)
    assert R.gn_pool_fwd_path(32, 33, 47) == ("generic", None)
    assert R.gn_pool_fwd_path(32, 34, 46) == ("slab", 2)       # 34 = 2 * 17: two-row slabs
    assert R.gn_pool_bwd_plan(64, 64, 32, 16) == (8, 8)         # config #2 stem: cluster of 8, 8-row slabs
    assert R.gn_pool_bwd_plan(16, 16, 32, 16) == (1, 16)
    assert R.gn_pool_bwd_plan(33, 47, 32, 16) is None
    assert R.gn_pool_bwd_plan(34, 46, 32, 16) is None           # 34 rows split over no power-of-two cluster
