"""CPU checks of the float64 recurrence reference that tests/test_gpu_recurrence.py judges the rnn.cu kernels by, and of
its error bars: the reference is torch.nn.LSTM / nn.GRU (forward and gradients) and the oracle's masked loop, the fp32
recurrence stays within every bar, and every perturbed reference misses it by at least 10x."""
import pytest
import torch

import rnn_reference as R
from oracle import torch_oracle as O


def _nn_and_ref(kind, T, n, H, D, seed):
    """an nn.LSTM / nn.GRU in float64 and the reference on its input projection, all masks true"""
    torch.manual_seed(seed)
    rnn = (torch.nn.LSTM if kind == "lstm" else torch.nn.GRU)(D, H).double()
    for name, p in rnn.named_parameters():
        torch.nn.init.orthogonal_(p) if "weight" in name else torch.nn.init.normal_(p, std=0.1)
    x = torch.randn(T, n, D, dtype=torch.float64, requires_grad=True)
    h0 = torch.tanh(torch.randn(n, H, dtype=torch.float64))
    c0 = torch.randn(n, H, dtype=torch.float64)
    dh_out = torch.randn(T, n, H, dtype=torch.float64)
    out, _ = rnn(x, (h0[None], c0[None]) if kind == "lstm" else h0[None])
    (out * dh_out).sum().backward()
    xproj = (x.detach() @ rnn.weight_ih_l0.detach().t() + rnn.bias_ih_l0.detach())
    ref = R.recurrence(kind, xproj, rnn.weight_hh_l0.detach(), rnn.bias_hh_l0.detach(), h0, c0,
                       torch.ones(T, n, dtype=torch.bool), dh_out)
    return rnn, x, out.detach(), h0, ref


@pytest.mark.parametrize("kind", ["lstm", "gru"])
def test_reference_is_torch_rnn(kind):
    """forward equals nn.LSTM / nn.GRU; dxproj (and dgh) chained through the input / recurrent GEMMs give nn's
    gradients of x, W_ih, W_hh and both biases"""
    T, n, H, D = 7, 5, 32, 24
    rnn, x, out, h0, ref = _nn_and_ref(kind, T, n, H, D, seed=3)
    tol = dict(rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(ref["hs"], out, **tol)
    dx = ref["dgates" if kind == "lstm" else "dgx"]
    dh = ref["dgates" if kind == "lstm" else "dgh"]
    h_in = torch.cat([h0[None], ref["hs"][:-1]], 0)
    torch.testing.assert_close(dx @ rnn.weight_ih_l0.detach(), x.grad, **tol)
    torch.testing.assert_close(torch.einsum("tng,tnd->gd", dx, x.detach()), rnn.weight_ih_l0.grad, **tol)
    torch.testing.assert_close(torch.einsum("tng,tnh->gh", dh, h_in), rnn.weight_hh_l0.grad, **tol)
    torch.testing.assert_close(dx.sum((0, 1)), rnn.bias_ih_l0.grad, **tol)
    torch.testing.assert_close(dh.sum((0, 1)), rnn.bias_hh_l0.grad, **tol)


@pytest.mark.parametrize("kind", ["lstm", "gru"])
def test_reference_is_oracle_masked_loop(kind):
    """with resets, the reference equals oracle.torch_oracle.rnn_seq_forward in float64"""
    T, n, H, D = 9, 6, 32, 16
    torch.manual_seed(5)
    G = 4 if kind == "lstm" else 3
    sd = {"rnn.weight_ih_l0": torch.randn(G * H, D, dtype=torch.float64) / D ** 0.5,
          "rnn.weight_hh_l0": torch.randn(G * H, H, dtype=torch.float64) / H ** 0.5,
          "rnn.bias_ih_l0": 0.1 * torch.randn(G * H, dtype=torch.float64),
          "rnn.bias_hh_l0": 0.1 * torch.randn(G * H, dtype=torch.float64)}
    x = torch.randn(T * n, D, dtype=torch.float64)
    masks = torch.rand(T * n, 1) > 0.25
    hidden = torch.randn(n, 2 if kind == "lstm" else 1, H, dtype=torch.float64)
    out, _ = O.rnn_seq_forward(x, hidden, masks, sd, "rnn.", kind.upper(), 1, n)
    xproj = (x @ sd["rnn.weight_ih_l0"].t() + sd["rnn.bias_ih_l0"]).view(T, n, G * H)
    ref = R.recurrence(kind, xproj, sd["rnn.weight_hh_l0"], sd["rnn.bias_hh_l0"], hidden[:, 0], hidden[:, -1],
                       masks.view(T, n))
    torch.testing.assert_close(ref["hs"].view(T * n, H), out, rtol=1e-12, atol=1e-13)


CPU_CASES = [("lstm", 1, 1, 32, "random", 1.0), ("lstm", 2, 8, 64, "random", 1.0), ("lstm", 48, 9, 32, "random", 1.0),
             ("lstm", 24, 33, 128, "chunk_bounds", 1.0), ("lstm", 16, 8, 256, "reset_t0", 1.0),
             ("lstm", 16, 9, 64, "random", 30.0), ("lstm", 2, 8, 32, "all_false", 1.0),
             ("gru", 1, 1, 32, "random", 1.0), ("gru", 2, 8, 64, "random", 1.0), ("gru", 48, 9, 32, "random", 1.0),
             ("gru", 24, 33, 128, "reset_last", 1.0), ("gru", 16, 8, 256, "all_true", 1.0),
             ("gru", 16, 9, 64, "random", 30.0), ("gru", 2, 8, 32, "all_false", 1.0)]


@pytest.mark.parametrize("kind,T,n,H,pattern,scale", CPU_CASES)
def test_bars_hold_fp32_and_catch_perturbations(kind, T, n, H, pattern, scale):
    """the fp32 recurrence (another summation order and other expf / tanhf) stays within every bar, and every
    perturbed reference that changes the result misses its bar by at least 10x"""
    c = R.make_case(kind, T, n, H, pattern, scale, seed=T + n + H)
    ref = R.recurrence(kind, **c)
    f32 = R.recurrence(kind, **c, dtype=torch.float32)
    ratios = {k: R.err_ratio(f32[k], ref[k], H) for k in ref}
    guards = R.guard_ratios(kind, c, ref, H)
    print(f"  {kind} T{T} n{n} H{H} {pattern} x{scale}: fp32 error / bar {ratios}; perturbed / bar {guards}")
    assert max(ratios.values()) <= 1.0, ratios
    assert guards and min(guards.values()) >= 10.0, guards
    expected = {"drop_b_hh"} | ({"bhn_outside_r", "dgh_without_r"} if kind == "gru" else set())
    assert expected <= guards.keys()   # these change every case
