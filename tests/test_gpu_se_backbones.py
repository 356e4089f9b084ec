"""GPU tests of the squeeze-excite backbones (se_resnet50 / se_resneXt50 / se_resneXt101, resnet.py:92-110, 155-180).

Kernel parity follows tests/test_gpu_deep_encoders.py: the reference is fp32 torch autograd on exactly the operands the
kernels read (fp16 y, bf16 g) with TF32 off, bars are scaled by the reference's max (check()), and each bar is shown to be
tight: a reference whose scale s has its last channel tile zeroed (forward), or whose squeeze gradient dp is dropped
(backward), or whose last channel tile is zeroed (excitation weight gradients) must miss it by at least 10x.
"""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_deep_encoders import _twice, bf, check, hf, zero_last_tile
from test_gpu_policy import _ODD_SPACES
from test_gpu_policy import test_encoder_any_size_any_keys as _encoder_vs_oracle
from test_gpu_policy import test_next_configs_vs_reference as _policy_vs_reference

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

DEV = "cuda"
G = 16   # GroupNorm groups of every policy backbone (ngroups = 16 at base planes 32)
# (C, hw) of the SE blocks at 256x256 input: layer1..layer4; then layer3 of a 62x30 input (2x1) and layer4 (1x1)
SE_SHAPES = [(128, 32 * 32), (256, 16 * 16), (512, 8 * 8), (1024, 4 * 4), (512, 2), (1024, 1)]
BATCHES = {"actor": 2, "learner": 1024}


@pytest.fixture(autouse=True)
def _no_tf32():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _gn_stats(y, groups):
    """the conv epilogue's GroupNorm statistics: f64 (sum, sumsq) per (frame, group) of NHWC y"""
    B, hw, C = y.shape
    v = y.double().view(B, hw, groups, C // groups)
    return torch.stack([v.sum((1, 3)), (v * v).sum((1, 3))], -1).contiguous()


def _case(C, hw, B, downsample, seed):
    """operands of one SE block output: y3 (and the downsample's pre-norm yd) fp16 NHWC with per-channel offsets, GN
    affines, excitation weights, and an upstream gradient with a per-(frame, channel) mean (so the squeeze's gradient
    dp is a visible part of dy)"""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device=DEV, generator=gen)  # noqa: E731
    cr = C // 16
    t = dict(
        y=hf(rn(B, hw, C) * (0.5 + rn(1, 1, C).abs()) + 0.5 * rn(1, 1, C)),
        gamma=1.0 + 0.3 * rn(C), beta=0.3 * rn(C),
        w1=rn(cr, C) / C ** 0.5, b1=0.1 * rn(cr), w2=rn(C, cr) / cr ** 0.5, b2=0.1 * rn(C),
        g=bf(rn(B, hw, C) + 2.0 * rn(B, 1, C)),
    )
    if downsample:
        t.update(yd=hf(rn(B, hw, C) + 0.2 * rn(1, 1, C)), gamma_d=1.0 + 0.3 * rn(C), beta_d=0.3 * rn(C))
    else:
        t["x"] = hf(torch.relu(rn(B, hw, C)))
    t["st"] = _gn_stats(t["y"], G)
    if downsample:
        t["st_d"] = _gn_stats(t["yd"], G)
    return t


def _gn(y, gamma, beta):
    B, hw, C = y.shape
    return F.group_norm(y.permute(0, 2, 1), G, gamma, beta, eps=1e-5).permute(0, 2, 1)


def _reference(t, s_zero_tile=False):
    """fp32 SEBottleneck tail on the kernels' operands: returns (p, s, pre-ReLU output, leaves)"""
    y = t["y"].float().requires_grad_(True)
    lv = {k: t[k].clone().requires_grad_(True) for k in ("gamma", "beta", "w1", "b1", "w2", "b2")}
    z = _gn(y, lv["gamma"], lv["beta"])
    p = z.mean(1)
    h = torch.relu(F.linear(p, lv["w1"], lv["b1"]))
    s = torch.sigmoid(F.linear(h, lv["w2"], lv["b2"]))
    if s_zero_tile:
        s = zero_last_tile(s)
    r = _gn(t["yd"].float(), t["gamma_d"], t["beta_d"]) if "yd" in t else t["x"].float()
    lv["y"] = y
    return p, h, s, s[:, None, :] * z + r, lv


def _run_fwd(hb, t, B, hw, C):
    from habitat_lab_b200 import ops

    cr = C // 16
    o = torch.empty(B, hw, C, dtype=torch.float16, device=DEV)
    ob = torch.empty(B, hw, C, dtype=torch.bfloat16, device=DEV)
    p, h, s = (torch.empty(B, n, device=DEV) for n in (C, cr, C))
    kw = dict(res_stats=t["st_d"], res_gamma=t["gamma_d"], res_beta=t["beta_d"]) if "yd" in t else {}

    def run():
        ops.gn_se_residual_relu(t["y"], t["st"], t["gamma"], t["beta"], t["yd"] if "yd" in t else t["x"], t["w1"],
                                t["b1"], t["w2"], t["b2"], p, h, s, o, B, hw, C, G, out_bf16=ob, **kw)

    return run, (o, ob, p, h, s)


def _run_bwd(hb, t, o, h, s, B, hw, C):
    from habitat_lab_b200 import ops

    cr = C // 16
    dy = torch.empty(B, hw, C, dtype=torch.bfloat16, device=DEV)
    gz = torch.empty_like(dy)
    dgamma, dbeta = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    a, dh = torch.empty(B, C, device=DEV), torch.empty(B, cr, device=DEV)
    dw1, db1 = torch.empty(cr, C, device=DEV), torch.empty(cr, device=DEV)
    dw2, db2 = torch.empty(C, cr, device=DEV), torch.empty(C, device=DEV)
    p = t["p"]

    def run():
        ops.gn_se_bwd(t["g"], o, t["y"], t["st"], t["gamma"], t["beta"], s, h, t["w1"], t["w2"], dgamma, dbeta, dy, gz,
                      a, dh, B, hw, C, G)
        ops.se_excite_wgrad(a, h, p, dh, dw1, db1, dw2, db2)

    return run, (dy, gz, dgamma, dbeta, a, dh, dw1, db1, dw2, db2)


@pytest.mark.parametrize("batch", list(BATCHES))
@pytest.mark.parametrize("res", ["identity", "downsample"])
@pytest.mark.parametrize("C,hw", SE_SHAPES, ids=lambda v: str(v))
def test_se_block_parity(hb, C, hw, res, batch):
    B = BATCHES[batch]
    t = _case(C, hw, B, res == "downsample", seed=C + hw + B)
    # ---- forward: o (fp16 and its bf16 twin), p, s
    run, (o, ob, p, h, s) = _run_fwd(hb, t, B, hw, C)
    run()
    torch.cuda.synchronize()
    p_ref, h_ref, s_ref, pre, lv = _reference(t)
    o_ref = torch.relu(pre).detach()
    o_bad = torch.relu(_reference(t, s_zero_tile=True)[3]).detach()
    # fp16 output rounding (2^-11 relative); s / p are fp32 sums of <= 1024 * 64 terms
    check("o", o.float(), o_ref, 2e-3, 2e-3, [o_bad])
    # the bf16 twin rounds the same fp32 value as o: both roundings apart at most
    torch.testing.assert_close(ob.float(), o.float(), rtol=2 ** -8 + 2 ** -11, atol=1e-6)
    check("p", p, p_ref.detach(), 1e-4, 1e-4, [zero_last_tile(p_ref.detach())])
    check("h", h, h_ref.detach(), 1e-4, 1e-4, [zero_last_tile(h_ref.detach())])
    check("s", s, s_ref.detach(), 1e-4, 1e-4, [zero_last_tile(s_ref.detach())])
    # ---- backward, through the kernel's own ReLU mask (o > 0) so that the mask is not a source of difference
    t["p"] = p
    runb, (dy, gz, dgamma, dbeta, a, dh, dw1, db1, dw2, db2) = _run_bwd(hb, t, o, h, s, B, hw, C)
    runb()
    torch.cuda.synchronize()
    gzr = t["g"].float() * (o.float() > 0)
    assert torch.equal(gz, bf(gzr))
    names = ("y", "gamma", "beta", "w1", "b1", "w2", "b2")
    ref = dict(zip(names, torch.autograd.grad(pre, [lv[k] for k in names], gzr)))
    # dp dropped: the squeeze is treated as a constant, so only s * gz reaches z
    y2 = t["y"].float().requires_grad_(True)
    ga2, be2 = t["gamma"].clone().requires_grad_(True), t["beta"].clone().requires_grad_(True)
    z2 = _gn(y2, ga2, be2)
    s2 = torch.sigmoid(F.linear(torch.relu(F.linear(z2.mean(1).detach(), t["w1"], t["b1"])), t["w2"], t["b2"]))
    nodp = dict(zip(("y", "gamma", "beta"), torch.autograd.grad(s2[:, None, :] * z2, [y2, ga2, be2], gzr)))
    # dy: bf16 output (2^-8 relative) of an fp32 GroupNorm backward
    check("dy", dy.float(), ref["y"], 1e-2, 5e-3, [nodp["y"]])
    check("dgamma", dgamma, ref["gamma"], 1e-3, 1e-3, [nodp["gamma"], zero_last_tile(ref["gamma"], 0)])
    check("dbeta", dbeta, ref["beta"], 1e-3, 1e-3, [nodp["beta"], zero_last_tile(ref["beta"], 0)])
    check("dW1", dw1, ref["w1"], 1e-3, 1e-3, [zero_last_tile(ref["w1"])])
    check("db1", db1, ref["b1"], 1e-3, 1e-3, [zero_last_tile(ref["b1"], 0)])
    check("dW2", dw2, ref["w2"], 1e-3, 1e-3, [zero_last_tile(ref["w2"], 0)])
    check("db2", db2, ref["b2"], 1e-3, 1e-3, [zero_last_tile(ref["b2"], 0)])


@pytest.mark.parametrize("C,hw", [(128, 32 * 32), (1024, 4 * 4)], ids=lambda v: str(v))
def test_se_kernels_are_run_to_run_identical(hb, C, hw):
    """both SE kernels and the excitation weight gradients: two launches on the main stream and one on a side stream
    give the same bits"""
    B = 1024
    t = _case(C, hw, B, True, seed=7 + C)
    run, outs = _run_fwd(hb, t, B, hw, C)
    o, ob, p, h, s = _twice(run, list(outs))
    t["p"] = p
    runb, outs_b = _run_bwd(hb, t, o, h, s, B, hw, C)
    _twice(runb, list(outs_b))


# ---------------------------------------------------------------------------------------------
# whole policies
# ---------------------------------------------------------------------------------------------
def test_se_resnet50_objectnav_vs_reference(hb):
    """SE-ResNet50 + GRU with config #3's sensors: state_dict layout, values / log-probs / entropy / hidden state, losses
    and per-tensor gradient norms (se.excite.* included, at the plain configs' bars) of one minibatch against what the
    real reference recorded"""
    _policy_vs_reference(hb, "ser50_objectnav")


def test_se_resnext50_imagenav_vs_reference(hb):
    """Config #4's SE-ResNeXt50 dual encoder + LSTM-2 against the real reference, at the plain configs' bars except for
    the gradient norms of se.excite.0.*: that gradient is dh p^T with dh = (W2^T a) * [h > 0] over the fixture's 8 frames,
    which cancels strongly at this small loss (value loss 0.05).  The fp16 / bf16 storage of the trunk moved those norms of two
    of the 32 SE blocks by 30-45 % on one H100 (both in layer1), while the median deviation of all SE norms was 0.7 %.  Those norms get
    a 0.6 bar and the median of the SE norms a 2 % bar; the SE kernels' own arithmetic is pinned by test_se_block_parity."""
    import sys
    sys.path.insert(0, __file__.rsplit("/", 1)[0] + "/golden")
    from helpers import load_golden, recipe_state_dict
    from recipe import objectnav_rollout
    from test_gpu_policy import _next_case_spaces

    G = load_golden("serx50_imagenav")
    c = G["case"]
    obs_space, act_space = _next_case_spaces(c)
    pol = hb.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, num_recurrent_layers=c["layers"], rnn_type=c["rnn"],
                                  resnet_baseplanes=32, backbone=c["backbone"], normalize_visual_inputs=True)
    assert {k: tuple(v.shape) for k, v in pol.state_dict().items()} == {k: tuple(v) for k, v in G["shapes"].items()}
    assert list(pol.net.visual_encoder.visual_keys) == list(G["visual_keys"])
    pol.load_state_dict(recipe_state_dict(G["shapes"], c["seed"]))
    pol.to(DEV).train()
    st = hb.RolloutStorage(c["T"], c["N"], obs_space, act_space, pol)
    bufs, next_value = objectnav_rollout(c["T"], c["N"], c["H"], c["W"], c["n_actions"], c["layers"] * 2, 512, c["seed"],
                                         c["n_categories"], c["imagegoal"])
    for k, v in bufs["observations"].items():
        st.buffers["observations"][k].copy_(v)
    for k in ("recurrent_hidden_states", "masks", "rewards", "value_preds", "returns", "action_log_probs", "actions",
              "prev_actions"):
        st.buffers[k].copy_(bufs[k])
    st.current_rollout_step_idxs = [c["T"]]
    st.to(DEV)
    st.compute_returns(next_value.to(DEV), True, 0.99, 0.95)
    torch.manual_seed(G["mb_env_inds_seed"])
    batch = next(iter(st.data_generator(G["advantages"].to(DEV), 1)))
    metrics = pol.loss_and_backward(batch, 0.2, 0.5, 0.01, True).cpu()
    torch.cuda.synchronize()
    last = pol._last
    assert (last["values"].cpu() - G["eval_values"].view(-1)).abs().max().item() < 5e-3
    assert (last["log_probs"].cpu() - G["eval_log_probs"].view(-1)).abs().max().item() < 5e-3
    assert (last["entropy"].cpu() - G["eval_entropy"].view(-1)).abs().max().item() < 5e-4
    assert (last["hidden_out"].cpu() - G["eval_hidden"]).abs().max().item() < 5e-3
    got = dict(value_loss=metrics[0].item(), action_loss=metrics[1].item(), dist_entropy=metrics[2].item(),
               total=metrics[10].item())
    for k in got:
        assert got[k] == pytest.approx(G["mb_losses"][k], rel=1e-3, abs=2e-4), (k, got[k], G["mb_losses"][k])
    bad, se_dev = [], []
    for k, prm in pol.named_parameters():
        gn_ref, gn = G["grad_norms"][k], prm.grad.norm().item()
        if ".se.excite.0." in k:
            tol = 0.6
        else:
            tol = (0.25 if prm.dim() == 1 else 0.15) if "encoder" in k else 2e-2
        if ".se." in k:
            se_dev.append(abs(gn - gn_ref) / gn_ref)
        if abs(gn - gn_ref) > tol * gn_ref + 1e-7:
            bad.append((k, gn, gn_ref))
    assert not bad, bad[:8]
    se_dev.sort()
    assert len(se_dev) == 128 and se_dev[len(se_dev) // 2] < 0.02, se_dev[len(se_dev) // 2]


@pytest.mark.parametrize("shapes", _ODD_SPACES)
@pytest.mark.parametrize("backbone", ["se_resnet50", "se_resneXt101"])
def test_se_encoder_any_size_vs_oracle(hb, shapes, backbone):
    _encoder_vs_oracle(hb, shapes, backbone)


def _se_policy(hb, backbone, H=256):
    from habitat_lab_b200 import synthetic as syn

    if backbone == "se_resnet50":
        obs_space, act_space = syn.objectnav_spaces(H, H, 6, 21)
        pol = hb.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, num_recurrent_layers=1, rnn_type="GRU",
                                      resnet_baseplanes=32, backbone=backbone, normalize_visual_inputs=True)
        return pol, obs_space, act_space, 6
    obs_space, act_space = syn.imagenav_spaces(H, H, 4)
    pol = hb.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, num_recurrent_layers=2, rnn_type="LSTM",
                                  resnet_baseplanes=32, backbone=backbone, normalize_visual_inputs=True)
    return pol, obs_space, act_space, 4


@pytest.mark.parametrize("backbone", ["se_resnet50", "se_resneXt50"])
def test_se_loss_and_backward_is_run_to_run_identical(hb, backbone):
    from habitat_lab_b200.synthetic import fill_rollout_

    torch.manual_seed(9)
    pol, obs_space, act_space, A = _se_policy(hb, backbone)
    pol.to(DEV).train()
    T, N = 16, 16   # 256 frames
    st = hb.RolloutStorage(T, N, obs_space, act_space, pol)
    st.to(DEV)
    nv = fill_rollout_(st, seed=9, observation_space=obs_space, n_actions=A)
    st.compute_returns(nv, True, 0.99, 0.95)
    ppo = hb.PPO(pol, clip_param=0.2, ppo_epoch=1, num_mini_batch=1, value_loss_coef=0.5, entropy_coef=0.01, lr=2.5e-4,
                 eps=1e-5, max_grad_norm=0.2, use_clipped_value_loss=True, use_normalized_advantage=False)
    adv = ppo.get_advantages(st)
    sd = {k: v.clone() for k, v in pol.state_dict().items()}
    runs = []
    for _ in range(2):
        pol.load_state_dict(sd)
        torch.manual_seed(77)
        batch = next(iter(st.data_generator(adv, 1)))
        m = pol.loss_and_backward(batch, 0.2, 0.5, 0.01, True).clone()
        torch.cuda.synchronize()
        runs.append((m, {n: p.grad.clone() for n, p in pol.named_parameters() if p.grad is not None}))
    (m1, g1), (m2, g2) = runs
    assert torch.equal(m1, m2)
    assert any(".se.excite." in n for n in g1)
    assert all(g1[n].abs().max().item() > 0 for n in g1 if ".se.excite." in n)
    differ = [n for n in g1 if not torch.equal(g1[n], g2[n])]
    assert not differ, f"gradients differ run to run: {differ}"


def test_se_graphed_actor_replays_act(hb):
    """act() of an SE policy, and its CUDA-graph replay, against eager act()"""
    from habitat_lab_b200.synthetic import fill_rollout_

    torch.manual_seed(5)
    pol, obs_space, act_space, A = _se_policy(hb, "se_resneXt50", H=128)
    pol.to(DEV).eval()
    T, N = 4, 8
    st = hb.RolloutStorage(T, N, obs_space, act_space, pol)
    st.to(DEV)
    fill_rollout_(st, seed=2, observation_space=obs_space, n_actions=A, p_done=0.2)
    ob = st.buffers["observations"]
    step = lambda t: ({k: v[t] for k, v in ob.items()}, st.buffers["recurrent_hidden_states"][t],  # noqa: E731
                      st.buffers["prev_actions"][t], st.buffers["masks"][t])
    ga = hb.GraphedActor(pol, *step(0), deterministic=True)
    for t in (1, 2):
        ref = pol.act(*step(t), deterministic=True)
        got = ga(*step(t))
        torch.cuda.synchronize()
        assert torch.equal(got.actions, ref.actions)
        torch.testing.assert_close(got.values, ref.values, rtol=0, atol=0)
        torch.testing.assert_close(got.rnn_hidden_states, ref.rnn_hidden_states, rtol=0, atol=0)
