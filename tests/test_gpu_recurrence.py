"""GPU parity of the LSTM / GRU recurrence kernels (csrc/rnn.cu) against a float64 reference, on every dispatch path.

The reference (tests/rnn_reference.py) runs the masked recurrence in float64 on the kernels' own fp32 operands, so the
input-projection GEMM is out of the comparison, and its backward is float64 autograd seeded with the same dh_out.  Every
output of every product entry point is compared: hs, cs, gates / saved forward; dgates, or dgx and dgh, backward; h_in
of rnn_shift_mask bit for bit.  Each output has one bar, K u sqrt(H) of the reference's max, from the error analysis
in rnn_reference.py, and each case also shows the bar is tight: references with a stale h_{t-1} in the last CTA, an
ignored reset, b_hh dropped (GRU: b_hn outside r), the recurrent dh path dropped at one step, dc unmasked at a reset,
a zeroed carry (GRU: dgh without r) must miss it by at least 10x.

Operands follow the product's layout: h0 / c0 are hid[:, l] views of an [n, 4, H] state and b_hh is passed to the
forward separately, as NativeNetPolicy._rnn_forward does.

Dispatch: lstm_seq_fwd runs the v1 kernel below H = 512 and when h0 is misaligned or its row stride is not a multiple
of 4, else v2; lstm_seq_bwd runs v1 below H = 512, v2 at 512; the GRU has one kernel per direction.
"""
import pytest
import torch

import rnn_reference as R
from test_gpu_deep_encoders import _twice

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

DEV = "cuda"
HIDDEN = (32, 64, 128, 256, 512)
NS = (1, 8, 31, 32, 33, 64)
TS = (1, 2, 128)

# (T, n, H, mask pattern, pre-activation scale); 30 saturates most gates
_SWEEP = [(T, n, H, "random", 1.0) for H in HIDDEN for n in NS for T in TS]
_PATTERNS = [(128, 33, H, p, 1.0) for H in (128, 512) for p in R.MASK_PATTERNS[1:]]
_SATURATED = [(128, 33, H, "random", 30.0) for H in (64, 512)]
LSTM_CASES = _SWEEP + [(T, 41, 512, "random", 1.0) for T in TS] + _PATTERNS + _SATURATED   # n = 41: v2's partial tile
GRU_CASES = _SWEEP + [(128, 33, H, p, 1.0) for H in (64, 512) for p in R.MASK_PATTERNS[1:]] + \
    [(128, 33, H, "random", 30.0) for H in (32, 512)]


def _ids(cases):
    return [f"T{T}-n{n}-H{H}-{p}" + ("-sat" if s != 1.0 else "") for T, n, H, p, s in cases]


def _ws():
    return torch.zeros(64, dtype=torch.uint8, device=DEV)


def _on_gpu(c, T, n, H):
    """the case's operands on the GPU: h0 / c0 as hid[:, 1] / hid[:, 3] of an [n, 4, H] state, u8 masks [T * n]"""
    hid = torch.zeros(n, 4, H, device=DEV)
    hid[:, 1] = c["h0"].to(DEV)
    hid[:, 3] = c["c0"].to(DEV)
    d = {k: c[k].to(DEV).contiguous() for k in ("xproj", "w_hh", "b_hh", "dh_out")}
    d.update(hid=hid, h0=hid[:, 1], c0=hid[:, 3], mk=c["masks"].reshape(-1).to(DEV).view(torch.uint8))
    return d


def _ref_ops(c):
    return {k: c[k].to(DEV) for k in ("xproj", "w_hh", "b_hh", "h0", "c0", "masks", "dh_out")}


def _lstm_fwd(d, T, n, H, h0, c0, with_gates=True):
    from habitat_lab_b200 import ops

    hs, cs = torch.empty(T, n, H, device=DEV), torch.empty(T, n, H, device=DEV)
    gates = torch.empty(T, n, 4 * H, device=DEV) if with_gates else None
    ops.lstm_seq_fwd(d["xproj"].view(T * n, 4 * H), d["w_hh"], d["b_hh"], d["mk"], h0, c0, hs, cs, gates, T, n, H,
                     _ws())
    return hs, cs, gates


def _gru_fwd(d, T, n, H, with_saved=True):
    from habitat_lab_b200 import ops

    hs = torch.empty(T, n, H, device=DEV)
    saved = torch.empty(T, n, 4 * H, device=DEV) if with_saved else None
    ops.gru_seq_fwd(d["xproj"].view(T * n, 3 * H), d["w_hh"], d["b_hh"], d["mk"], d["h0"], hs, saved, T, n, H, _ws())
    return hs, saved


def _check(kind, got, ref, ops_, H, label):
    ratios = {k: R.err_ratio(got[k], ref[k], H) for k in got}
    guards = R.guard_ratios(kind, ops_, ref, H)
    print(f"  {label}: error / bar {({k: round(v, 3) for k, v in ratios.items()})}; "
          f"perturbed / bar {({k: round(v) for k, v in guards.items()})}")
    for k, r in ratios.items():
        assert torch.isfinite(got[k]).all(), f"{k}: not finite"
        assert r <= 1.0, f"{k}: error {r:.3f}x the bar"
    for p, g in guards.items():
        assert g >= 10.0, f"perturbation {p} only misses the bar by {g:.2f}x"


def _check_shift_mask(d, hs, T, n, H):
    from habitat_lab_b200 import ops

    hin = torch.full((T, n, H), float("nan"), device=DEV)
    ops.rnn_shift_mask(hs, d["h0"], d["mk"], hin, T, n, H)
    prev = torch.cat([d["h0"].unsqueeze(0), hs[:-1]], 0)
    ref = torch.where(d["mk"].view(T, n, 1).bool(), prev, torch.zeros((), device=DEV))
    assert torch.equal(hin, ref)


@pytest.mark.parametrize("T,n,H,pattern,scale", LSTM_CASES, ids=_ids(LSTM_CASES))
def test_lstm_recurrence(hb, T, n, H, pattern, scale):
    from habitat_lab_b200 import ops

    c = R.make_case("lstm", T, n, H, pattern, scale, seed=T * 1000 + n * 10 + H)
    d = _on_gpu(c, T, n, H)
    hs, cs, gates = _lstm_fwd(d, T, n, H, d["h0"], d["c0"])
    dg = torch.empty(T, n, 4 * H, device=DEV)
    ops.lstm_seq_bwd(d["dh_out"], gates, cs, d["c0"], d["w_hh"], d["mk"], dg, T, n, H, _ws())
    torch.cuda.synchronize()
    ops_ = _ref_ops(c)
    ref = R.recurrence("lstm", **ops_)
    _check("lstm", dict(hs=hs, cs=cs, gates=gates, dgates=dg), ref, ops_, H,
           f"lstm T{T} n{n} H{H} {pattern} x{scale:g}")
    _check_shift_mask(d, hs, T, n, H)


@pytest.mark.parametrize("T,n,H,pattern,scale", GRU_CASES, ids=_ids(GRU_CASES))
def test_gru_recurrence(hb, T, n, H, pattern, scale):
    from habitat_lab_b200 import ops

    c = R.make_case("gru", T, n, H, pattern, scale, seed=T * 1000 + n * 10 + H + 1)
    d = _on_gpu(c, T, n, H)
    hs, saved = _gru_fwd(d, T, n, H)
    dgx, dgh = torch.empty(T, n, 3 * H, device=DEV), torch.empty(T, n, 3 * H, device=DEV)
    ops.gru_seq_bwd(d["dh_out"], saved, hs, d["h0"], d["w_hh"], d["mk"], dgx, dgh, T, n, H, _ws())
    torch.cuda.synchronize()
    ops_ = _ref_ops(c)
    ref = R.recurrence("gru", **ops_)
    _check("gru", dict(hs=hs, saved=saved, dgx=dgx, dgh=dgh), ref, ops_, H,
           f"gru T{T} n{n} H{H} {pattern} x{scale:g}")
    _check_shift_mask(d, hs, T, n, H)


@pytest.mark.parametrize("T,n", [(2, 8), (128, 33)])
def test_lstm_fwd_v1_at_512(hb, T, n):
    """h0 / c0 with row stride 513 (not a multiple of 4) send H = 512 to the v1 forward kernel: it must match the
    reference and the v2 kernel (contiguous h0 / c0) within the bars"""
    H = 512
    c = R.make_case("lstm", T, n, H, seed=T + n)
    d = _on_gpu(c, T, n, H)
    bufs = [torch.zeros(n, H + 1, device=DEV) for _ in range(2)]
    bufs[0][:, :H] = d["h0"]
    bufs[1][:, :H] = d["c0"]
    v1 = _lstm_fwd(d, T, n, H, bufs[0][:, :H], bufs[1][:, :H])
    v2 = _lstm_fwd(d, T, n, H, d["h0"].contiguous(), d["c0"].contiguous())
    torch.cuda.synchronize()
    ops_ = _ref_ops(c)
    ops_["dh_out"] = None
    ref = R.recurrence("lstm", **ops_)
    names = ("hs", "cs", "gates")
    _check("lstm", dict(zip(names, v1)), ref, ops_, H, f"lstm v1 at 512, T{T} n{n}")
    for k, a, b in zip(names, v1, v2):
        assert R.err_ratio(a, b, H) <= 1.0, k


@pytest.mark.parametrize("kind", ["lstm", "gru"])
@pytest.mark.parametrize("n", [64, 512])
def test_actor_step_without_saved_gates(hb, kind, n):
    """the actor's step (T = 1, gates_out / saved = NULL) writes the same bits as the training launch"""
    T, H = 1, 512
    c = R.make_case(kind, T, n, H, seed=n)
    d = _on_gpu(c, T, n, H)
    if kind == "lstm":
        with_g, without = _lstm_fwd(d, T, n, H, d["h0"], d["c0"]), _lstm_fwd(d, T, n, H, d["h0"], d["c0"], False)
        got = dict(hs=without[0], cs=without[1])
        assert torch.equal(with_g[0], without[0]) and torch.equal(with_g[1], without[1])
    else:
        with_g, without = _gru_fwd(d, T, n, H), _gru_fwd(d, T, n, H, False)
        got = dict(hs=without[0])
        assert torch.equal(with_g[0], without[0])
    torch.cuda.synchronize()
    ops_ = _ref_ops(c)
    ops_["dh_out"] = None
    _check(kind, got, R.recurrence(kind, **ops_), ops_, H, f"{kind} actor n{n}")


def _chunked_bwd(d, gates, cs, T, n, H, C, dg, carry):
    from habitat_lab_b200 import ops

    Tc = T // C
    for ci in reversed(range(C)):
        t0, t1 = ci * Tc, (ci + 1) * Tc
        c0 = d["c0"] if ci == 0 else cs[t0 - 1]
        ops.lstm_seq_bwd_chunk(d["dh_out"][t0:t1], gates[t0:t1], cs[t0:t1], c0, d["w_hh"], d["mk"][t0 * n:t1 * n],
                               dg[t0:t1], Tc, n, H, _ws(), carry, carry_in=ci < C - 1, carry_out=ci > 0)


@pytest.mark.parametrize("n", [8, 33])
@pytest.mark.parametrize("C", [2, 4, 32])
def test_lstm_time_chunks_are_exact(hb, n, C):
    """lstm_seq_fwd over C time chunks (h0 / c0 = the previous chunk's last rows) and lstm_seq_bwd_chunk walked last to
    first with the carry give the one-launch results bit for bit; C = 32 is one step per chunk (carry_out at t = 0)"""
    from habitat_lab_b200 import ops

    T, H = 32, 512
    Tc = T // C
    c = R.make_case("lstm", T, n, H, "chunk_bounds", seed=n + C)
    c["masks"][:, 0] = True   # one sequence runs across every chunk boundary
    d = _on_gpu(c, T, n, H)
    hs, cs, gates = _lstm_fwd(d, T, n, H, d["h0"], d["c0"])
    hs2, cs2, gates2 = (torch.full_like(t, float("nan")) for t in (hs, cs, gates))
    for ci in range(C):
        t0, t1 = ci * Tc, (ci + 1) * Tc
        h0 = d["h0"] if ci == 0 else hs2[t0 - 1]
        c0 = d["c0"] if ci == 0 else cs2[t0 - 1]
        ops.lstm_seq_fwd(d["xproj"].view(T * n, 4 * H)[t0 * n:t1 * n], d["w_hh"], d["b_hh"], d["mk"][t0 * n:t1 * n],
                         h0, c0, hs2[t0:t1], cs2[t0:t1], gates2[t0:t1], Tc, n, H, _ws())
    dg = torch.empty(T, n, 4 * H, device=DEV)
    ops.lstm_seq_bwd(d["dh_out"], gates, cs, d["c0"], d["w_hh"], d["mk"], dg, T, n, H, _ws())
    dg2 = torch.full_like(dg, float("nan"))
    _chunked_bwd(d, gates, cs, T, n, H, C, dg2, torch.full((2, n, H), float("nan"), device=DEV))
    torch.cuda.synchronize()
    for a, b in ((hs, hs2), (cs, cs2), (gates, gates2), (dg, dg2)):
        assert torch.equal(a, b)


RTR_KERNELS = ["lstm_fwd_v1", "lstm_fwd_v1_512", "lstm_fwd_v2", "lstm_bwd_v1", "lstm_bwd_v2", "lstm_bwd_chunk",
               "gru_fwd", "gru_bwd", "shift_mask"]


@pytest.mark.parametrize("kernel", RTR_KERNELS)
def test_recurrence_is_run_to_run_identical(hb, kernel):
    """each product recurrence launch twice on the main stream and once on a side stream: bit-identical outputs"""
    from habitat_lab_b200 import ops

    T, n = 32, 33
    H = 128 if kernel in ("lstm_fwd_v1", "lstm_bwd_v1") else 512
    kind = "gru" if kernel.startswith("gru") else "lstm"
    c = R.make_case(kind, T, n, H, seed=len(kernel))
    d = _on_gpu(c, T, n, H)
    if kind == "gru":
        hs, saved = _gru_fwd(d, T, n, H)
        if kernel == "gru_fwd":
            outs = [hs, saved]
            _twice(lambda: ops.gru_seq_fwd(d["xproj"].view(T * n, 3 * H), d["w_hh"], d["b_hh"], d["mk"], d["h0"], hs,
                                           saved, T, n, H, _ws()), outs)
        else:
            outs = [torch.empty(T, n, 3 * H, device=DEV) for _ in range(2)]
            _twice(lambda: ops.gru_seq_bwd(d["dh_out"], saved, hs, d["h0"], d["w_hh"], d["mk"], *outs, T, n, H, _ws()),
                   outs)
        return
    hs, cs, gates = _lstm_fwd(d, T, n, H, d["h0"], d["c0"])
    if kernel.startswith("lstm_fwd"):
        h0, c0 = d["h0"], d["c0"]
        if kernel == "lstm_fwd_v1_512":
            bufs = [torch.zeros(n, H + 1, device=DEV) for _ in range(2)]
            bufs[0][:, :H], bufs[1][:, :H] = h0, c0
            h0, c0 = bufs[0][:, :H], bufs[1][:, :H]
        outs = [hs, cs, gates]
        _twice(lambda: ops.lstm_seq_fwd(d["xproj"].view(T * n, 4 * H), d["w_hh"], d["b_hh"], d["mk"], h0, c0, *outs,
                                        T, n, H, _ws()), outs)
    elif kernel == "lstm_bwd_chunk":
        outs = [torch.empty(T, n, 4 * H, device=DEV), torch.empty(2, n, H, device=DEV)]
        _twice(lambda: _chunked_bwd(d, gates, cs, T, n, H, 4, *outs), outs)
    elif kernel.startswith("lstm_bwd"):
        outs = [torch.empty(T, n, 4 * H, device=DEV)]
        _twice(lambda: ops.lstm_seq_bwd(d["dh_out"], gates, cs, d["c0"], d["w_hh"], d["mk"], outs[0], T, n, H, _ws()),
               outs)
    else:
        outs = [torch.empty(T, n, H, device=DEV)]
        _twice(lambda: ops.rnn_shift_mask(hs, d["h0"], d["mk"], outs[0], T, n, H), outs)


@pytest.mark.parametrize("kind,H", [("lstm", 128), ("lstm", 512), ("gru", 128)])
def test_misaligned_backward_buffer_is_an_argument_error(hb, kind, H):
    """dgates / dgh are read back with 16-byte loads: a pointer 4 bytes off is refused before any launch"""
    from habitat_lab_b200 import ops

    T, n = 2, 8
    c = R.make_case(kind, T, n, H, seed=H)
    d = _on_gpu(c, T, n, H)
    G = 4 if kind == "lstm" else 3
    buf = torch.zeros(T * n * G * H + 4, device=DEV)
    bad = buf[1:1 + T * n * G * H].view(T, n, G * H)
    assert bad.data_ptr() % 16 == 4
    if kind == "lstm":
        hs, cs, gates = _lstm_fwd(d, T, n, H, d["h0"], d["c0"])

        def call():
            ops.lstm_seq_bwd(d["dh_out"], gates, cs, d["c0"], d["w_hh"], d["mk"], bad, T, n, H, _ws())
    else:
        hs, saved = _gru_fwd(d, T, n, H)
        dgx = torch.empty(T, n, 3 * H, device=DEV)

        def call():
            ops.gru_seq_bwd(d["dh_out"], saved, hs, d["h0"], d["w_hh"], d["mk"], dgx, bad, T, n, H, _ws())
    torch.cuda.synchronize()
    lib = hb.load()
    before = lib.hb200_launch_count()
    with pytest.raises(hb.Hb200Error, match="16-byte aligned"):
        call()
    assert lib.hb200_launch_count() == before
    torch.cuda.synchronize()


def test_wavefront_loss_and_backward_is_run_to_run_identical(hb):
    """config #2 (LSTM-512 x 2) at T = 32: the two layers run as a wavefront on two streams, forward and backward;
    the same minibatch twice from the same state gives the same metrics and gradients bit for bit"""
    from habitat_lab_b200.synthetic import fill_rollout_, pointnav_spaces

    T, N = 32, 32
    torch.manual_seed(2)
    obs_space, act_space = pointnav_spaces(64, 64)
    pol = hb.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, num_recurrent_layers=2, rnn_type="LSTM",
                                  resnet_baseplanes=32, backbone="resnet18", normalize_visual_inputs=True).to(DEV)
    pol.train()
    assert pol._rnn_wavefront(True, 512, 2, T)
    st = hb.RolloutStorage(T, N, obs_space, act_space, pol)
    st.to(DEV)
    nv = fill_rollout_(st, seed=2, p_done=0.1)
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
        runs.append((m, {k: p.grad.clone() for k, p in pol.named_parameters() if p.grad is not None}))
    (m1, g1), (m2, g2) = runs
    assert torch.equal(m1, m2)
    assert g1.keys() == g2.keys() and len(g1) > 0
    differ = [k for k in g1 if not torch.equal(g1[k], g2[k])]
    assert not differ, f"gradients differ run to run: {differ}"
