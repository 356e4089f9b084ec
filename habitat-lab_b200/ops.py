"""Thin typed wrappers over the C ABI (include/hb200.h): torch tensors in, device pointers
out.  torch is plumbing only (allocation, streams); every computation happens in libhb200.so."""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import ConvShape, call, load, ptr

BF16 = torch.bfloat16
F16 = torch.float16
N_METRICS = 12
METRIC_KEYS = ("value_loss", "action_loss", "dist_entropy", "value_pred_min", "value_pred_mean",
               "value_pred_max", "prob_ratio_min", "prob_ratio_mean", "prob_ratio_max",
               "ppo_fraction_clipped", "total_loss")


def _chk(t: torch.Tensor, dtype, name: str):
    if not t.is_cuda:
        raise _lib.Hb200Error(f"{name}: expected a CUDA tensor (no CPU fallback)")
    if t.dtype != dtype:
        raise _lib.Hb200Error(f"{name}: expected {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise _lib.Hb200Error(f"{name}: expected a contiguous tensor")


def as_u8(masks: torch.Tensor) -> torch.Tensor:
    return masks.view(torch.uint8) if masks.dtype == torch.bool else masks


# ---- GAE / advantages ---------------------------------------------------------------------
def gae_adv(rewards, value_preds, masks, next_value, returns, advantages, stats, t_cur, gamma, tau,
            use_gae=True, variant=0):
    t_alloc, n = rewards.shape[0], rewards.shape[1]
    for t, nm in ((rewards, "rewards"), (value_preds, "value_preds"), (returns, "returns"), (next_value, "next_value")):
        _chk(t, torch.float32, nm)
    call("hb200_gae_adv", ptr(rewards), ptr(value_preds), ptr(as_u8(masks)), ptr(next_value), ptr(returns),
         ptr(advantages), ptr(stats), int(t_cur), int(t_alloc), int(n), float(gamma), float(tau),
         int(bool(use_gae)), int(variant))


def adv_normalize(advantages, stats=None, mean_var=None):
    mode = 0 if mean_var is None else 1
    call("hb200_adv_normalize", ptr(advantages), advantages.numel(), ptr(stats), ptr(mean_var), mode)


# ---- heads + loss ---------------------------------------------------------------------------
def ppo_loss_workspace(batch, hidden, n_actions, device):
    nbytes = load().hb200_ppo_loss_workspace_bytes(batch, hidden, n_actions)
    return torch.empty(nbytes, dtype=torch.uint8, device=device)


def ppo_loss(features, w_act, b_act, w_val, b_val, actions, old_lp, adv, old_v, returns, clip, c_v, c_e,
             use_clipped_value_loss, compute_grads, out, workspace, is_coeffs=None):
    """out: dict with optional tensors values/log_probs/entropy, d_features, d_w_act, d_b_act,
    d_w_val, d_b_val, metrics."""
    B, H = features.shape
    A = w_act.shape[0]
    _chk(features, torch.float32, "features")
    _chk(actions, torch.int64, "actions")
    call("hb200_ppo_loss", ptr(features), ptr(w_act), ptr(b_act), ptr(w_val), ptr(b_val), ptr(actions),
         ptr(old_lp), ptr(adv), ptr(old_v), ptr(returns), ptr(is_coeffs), B, H, A, float(clip), float(c_v),
         float(c_e), int(bool(use_clipped_value_loss)), int(bool(compute_grads)),
         ptr(out.get("values")), ptr(out.get("log_probs")), ptr(out.get("entropy")),
         ptr(out.get("d_features")), ptr(out.get("d_w_act")), ptr(out.get("d_b_act")),
         ptr(out.get("d_w_val")), ptr(out.get("d_b_val")), ptr(out["metrics"]), ptr(workspace))


# ---- optimizer ----------------------------------------------------------------------------------
def clip_adam_workspace(n, device):
    return torch.empty(load().hb200_clip_adam_workspace_bytes(n), dtype=torch.uint8, device=device)


def clip_adam(params, grads, exp_avg, exp_avg_sq, lr, betas, eps, weight_decay, max_grad_norm, grad_scale,
              step, grad_norm_out, workspace, hyper=None):
    for t, nm in ((params, "params"), (grads, "grads"), (exp_avg, "exp_avg"), (exp_avg_sq, "exp_avg_sq")):
        _chk(t, torch.float32, nm)
    call("hb200_clip_adam", ptr(params), ptr(grads), ptr(exp_avg), ptr(exp_avg_sq), params.numel(), float(lr),
         float(betas[0]), float(betas[1]), float(eps), float(weight_decay),
         float(max_grad_norm if max_grad_norm is not None else 0.0), float(grad_scale), int(step), ptr(hyper),
         ptr(grad_norm_out), ptr(workspace))


# ---- visual prep ------------------------------------------------------------------------------------
def prep_stats(rgb, depth, frame_rows, H, W, stats_acc, rgb_scale=1.0 / 255.0):
    call("hb200_prep_stats", ptr(rgb), ptr(depth), ptr(frame_rows), frame_rows.numel(), H, W,
         3 if rgb is not None else 0, 1 if depth is not None else 0, float(rgb_scale), ptr(stats_acc))


def prep_finalize(stats_acc, run_mean, run_var, run_count, scale_shift, channels, pixels_per_frame, update):
    call("hb200_prep_finalize", ptr(stats_acc), ptr(run_mean), ptr(run_var), ptr(run_count), ptr(scale_shift),
         channels, int(pixels_per_frame), int(bool(update)))


def prep_apply(rgb, depth, frame_rows, H, W, scale_shift, out, rgb_scale=1.0 / 255.0, s2d=False, out_bf16=None):
    call("hb200_prep_apply", ptr(rgb), ptr(depth), ptr(frame_rows), frame_rows.numel(), H, W,
         3 if rgb is not None else 0, 1 if depth is not None else 0, float(rgb_scale), ptr(scale_shift), ptr(out),
         ptr(out_bf16), int(bool(s2d)))


# ---- conv ----------------------------------------------------------------------------------------------
def conv_shape(batch, hi, wi, ci, co, kh, kw, stride, pad) -> ConvShape:
    ho = (hi + 2 * pad - kh) // stride + 1
    wo = (wi + 2 * pad - kw) // stride + 1
    return ConvShape(batch, hi, wi, ci, ho, wo, co, kh, kw, stride, pad)


def packed_weight_elems(n_rows, k_channels, kh, kw) -> int:
    return load().hb200_packed_weight_elems(n_rows, k_channels, kh, kw)


def pack_conv_weight(w_oihw: torch.Tensor, ci_pad: int, want_t: bool = True):
    co, ci_real, kh, kw = w_oihw.shape
    _chk(w_oihw, torch.float32, "w_oihw")
    dev = w_oihw.device
    wp = torch.empty(packed_weight_elems(co, ci_pad, kh, kw), dtype=F16, device=dev)   # forward image: fp16
    wt = torch.empty(packed_weight_elems(ci_pad, co, kh, kw), dtype=BF16, device=dev) if want_t else None
    call("hb200_pack_conv_weight", ptr(w_oihw), ptr(wp), ptr(wt), co, ci_real, ci_pad, kh, kw)
    return wp, wt


def pack_conv_weight_into(w_oihw, wp, wt, ci_pad):
    co, ci_real, kh, kw = w_oihw.shape
    call("hb200_pack_conv_weight", ptr(w_oihw), ptr(wp), ptr(wt), co, ci_real, ci_pad, kh, kw)


def conv_fwd(x, wp, y, s: ConvShape, gn_stats=None, gn_groups=0):
    call("hb200_conv_fwd", ptr(x), ptr(wp), ptr(y), ptr(gn_stats), int(gn_groups), ctypes.addressof(s))


def conv_bias_act_fwd(x, wp, bias, y, s: ConvShape, relu):
    call("hb200_conv_bias_act_fwd", ptr(x), ptr(wp), ptr(bias), ptr(y), int(bool(relu)), ctypes.addressof(s))


def prep_plain(rgb, depth, frame_rows, H, W, c_rgb, c_depth, out):
    call("hb200_prep_plain", ptr(rgb), ptr(depth), ptr(frame_rows), frame_rows.numel(), H, W, c_rgb, c_depth, ptr(out))


def relu_bias_bwd(g, out, dy, dbias, npix, channels):
    call("hb200_relu_bias_bwd", ptr(g), ptr(out), ptr(dy), ptr(dbias), int(npix), channels)


def bf16_hwc_to_f32_chw(x, out, batch, hw, channels):
    call("hb200_bf16_hwc_to_f32_chw", ptr(x), ptr(out), batch, hw, channels)


def conv_dgrad(dy, wt, dx, s: ConvShape, addend=None):
    call("hb200_conv_dgrad", ptr(dy), ptr(wt), ptr(addend), ptr(dx), ctypes.addressof(s))


def conv_wgrad(x, dy, dw_acc, s: ConvShape):
    call("hb200_conv_wgrad", ptr(x), ptr(dy), ptr(dw_acc), ctypes.addressof(s))


def unpack_conv_wgrad(dw_acc, dw_oihw, ci_pad):
    co, ci_real, kh, kw = dw_oihw.shape
    call("hb200_unpack_conv_wgrad", ptr(dw_acc), ptr(dw_oihw), co, ci_real, ci_pad, kh, kw)


def conv_halo_supported(c, n, k, h, w) -> bool:
    return bool(load().hb200_conv_halo_supported(c, n, k, h, w))


def conv_halo_wgrad_supported(c, n, k, h, w) -> bool:
    return bool(load().hb200_conv_halo_wgrad_supported(c, n, k, h, w))


def pack_halo_weight(w_oihw, img, c, n, k, mode):
    co, ci_real = w_oihw.shape[0], w_oihw.shape[1]
    call("hb200_pack_halo_weight", ptr(w_oihw), ptr(img), co, ci_real, c, n, k, mode)


def conv_halo(x, wimg, y, batch, h, w, c, n, k, mode, addend=None, gn_stats=None, gn_groups=0):
    call("hb200_conv_halo", ptr(x), ptr(wimg), ptr(y), ptr(addend), ptr(gn_stats), int(gn_groups), batch, h, w, c, n,
         k, mode)


def conv_s2_supported(c, na, nb, h, w) -> bool:
    return bool(load().hb200_conv_s2_supported(int(c), int(na), int(nb), int(h), int(w)))


def conv_s2_fwd(x, wimg, ya, yb, batch, h, w, c, na, nb, stats_a=None, groups_a=0, stats_b=None, groups_b=0):
    """3x3 stride-2 conv (ya) + 1x1 stride-2 downsample conv (yb) of the same input in one launch (csrc/conv_s2.cu)"""
    call("hb200_conv_s2_fwd", ptr(x), ptr(wimg), ptr(ya), ptr(yb), ptr(stats_a), int(groups_a), ptr(stats_b),
         int(groups_b), batch, h, w, c, na, nb)


def conv_s2_wgrad_supported(c, n, h, w) -> bool:
    return bool(load().hb200_conv_s2_wgrad_supported(int(c), int(n), int(h), int(w)))


def conv_s2_wgrad(x_bf16, dy, dw_acc, batch, h, w, c, n):
    """dw_acc f32 [16*c, n] (pre-zeroed): weight gradient of the 3x3 stride-2 conv over the space-to-depth view"""
    call("hb200_conv_s2_wgrad", ptr(x_bf16), ptr(dy), ptr(dw_acc), batch, h, w, c, n)


def unpack_s2_wgrad(dw_acc, dw_oihw):
    call("hb200_unpack_s2_wgrad", ptr(dw_acc), ptr(dw_oihw), dw_oihw.shape[0], dw_oihw.shape[1])


def conv_s2_dgrad(dya, dyb, wimg_t, dx, batch, h, w, c, na, nb, addend=None):
    call("hb200_conv_s2_dgrad", ptr(dya), ptr(dyb), ptr(wimg_t), ptr(addend), ptr(dx), batch, h, w, c, na, nb)


def conv_halo_wgrad(x, dy, dw_acc, batch, h, w, c, n, k):
    call("hb200_conv_halo_wgrad", ptr(x), ptr(dy), ptr(dw_acc), batch, h, w, c, n, k)


def unpack_stem_wgrad(dw_acc, dw_oihw):
    call("hb200_unpack_stem_wgrad", ptr(dw_acc), ptr(dw_oihw), dw_oihw.shape[0], dw_oihw.shape[1])


def umma_gemm_probe(a, b, d, m, n, k, layout):
    call("hb200_umma_gemm_probe", ptr(a), ptr(b), ptr(d), m, n, k, layout)


# ---- GroupNorm & friends -----------------------------------------------------------------------------
def gn_apply(y, stats, gamma, beta, out, batch, hw, channels, groups, relu, eps=1e-5, chw_flat=False, out_bf16=None):
    mode = 0 if out.dtype != torch.float32 else (2 if chw_flat else 1)
    call("hb200_gn_apply", ptr(y), ptr(stats), ptr(gamma), ptr(beta), ptr(out), ptr(out_bf16), mode, batch, hw,
         channels, groups, float(eps), int(bool(relu)))


def gn_residual_relu(y, stats, gamma, beta, res, out, batch, hw, channels, groups, res_stats=None,
                     res_gamma=None, res_beta=None, eps=1e-5, out_bf16=None):
    call("hb200_gn_residual_relu", ptr(y), ptr(stats), ptr(gamma), ptr(beta), ptr(res), ptr(res_stats),
         ptr(res_gamma), ptr(res_beta), ptr(out), ptr(out_bf16), batch, hw, channels, groups, float(eps))


def gn_relu_maxpool(y, stats, gamma, beta, out, argmax, batch, h, w, channels, groups, eps=1e-5, out_bf16=None):
    call("hb200_gn_relu_maxpool", ptr(y), ptr(stats), ptr(gamma), ptr(beta), ptr(out), ptr(out_bf16), ptr(argmax),
         batch, h, w, channels, groups, float(eps))


def gn_relu_maxpool_bwd_supported(h, w, channels, groups) -> bool:
    return bool(load().hb200_gn_relu_maxpool_bwd_supported(h, w, channels, groups))


def gn_relu_maxpool_bwd(dpool, argmax, y, stats, gamma, beta, dgamma, dbeta, dy, batch, h, w, channels, groups,
                        eps=1e-5):
    call("hb200_gn_relu_maxpool_bwd", ptr(dpool), ptr(argmax), ptr(y), ptr(stats), ptr(gamma), ptr(beta), ptr(dgamma),
         ptr(dbeta), ptr(dy), batch, h, w, channels, groups, float(eps))


def maxpool_bwd(dout, argmax, dz, batch, h, w, channels):
    call("hb200_maxpool_bwd", ptr(dout), ptr(argmax), ptr(dz), batch, h, w, channels)


def gn_bwd_reduce(g, act, y, stats, gamma, beta, sums, dgamma, dbeta, batch, hw, channels, groups, mask_mode,
                  eps=1e-5):
    call("hb200_gn_bwd_reduce", ptr(g), ptr(act), ptr(y), ptr(stats), ptr(gamma), ptr(beta), ptr(sums),
         ptr(dgamma), ptr(dbeta), batch, hw, channels, groups, float(eps), mask_mode)


def gn_bwd_apply(g, act, y, stats, gamma, beta, sums, dy, gz_out, batch, hw, channels, groups, mask_mode,
                 eps=1e-5):
    call("hb200_gn_bwd_apply", ptr(g), ptr(act), ptr(y), ptr(stats), ptr(gamma), ptr(beta), ptr(sums), ptr(dy),
         ptr(gz_out), batch, hw, channels, groups, float(eps), mask_mode)


def gn_bwd(g, act, y, stats, gamma, beta, dgamma, dbeta, dy, gz_out, batch, hw, channels, groups, mask_mode, eps=1e-5):
    call("hb200_gn_bwd", ptr(g), ptr(act), ptr(y), ptr(stats), ptr(gamma), ptr(beta), ptr(dgamma), ptr(dbeta),
         ptr(dy), ptr(gz_out), batch, hw, channels, groups, float(eps), mask_mode)


def gn_se_residual_relu(y, stats, gamma, beta, res, w1, b1, w2, b2, p, h, s, out, batch, hw, channels, groups,
                        res_stats=None, res_gamma=None, res_beta=None, eps=1e-5, out_bf16=None):
    """out = relu(SE(GN(y)) + res); p / h / s f32 [B,C] / [B,C/16] / [B,C] are kept for gn_se_bwd (see hb200.h)"""
    call("hb200_gn_se_residual_relu", ptr(y), ptr(stats), ptr(gamma), ptr(beta), ptr(res), ptr(res_stats),
         ptr(res_gamma), ptr(res_beta), ptr(w1), ptr(b1), ptr(w2), ptr(b2), ptr(p), ptr(h), ptr(s), ptr(out),
         ptr(out_bf16), batch, hw, channels, groups, w1.shape[0], float(eps))


def gn_se_bwd(g, act, y, stats, gamma, beta, s, h, w1, w2, dgamma, dbeta, dy, gz_out, a, dh, batch, hw, channels,
              groups, eps=1e-5):
    call("hb200_gn_se_bwd", ptr(g), ptr(act), ptr(y), ptr(stats), ptr(gamma), ptr(beta), ptr(s), ptr(h), ptr(w1),
         ptr(w2), ptr(dgamma), ptr(dbeta), ptr(dy), ptr(gz_out), ptr(a), ptr(dh), batch, hw, channels, groups,
         w1.shape[0], float(eps))


def se_excite_wgrad(a, h, p, dh, dw1, db1, dw2, db2):
    """excitation weight gradients from gn_se_bwd's a / dh and the forward's p / h: dw2 = a^T h, db2 = sum_B a,
    dw1 = dh^T p, db1 = sum_B dh (fp32 GEMMs and column sums in a fixed order; written, not accumulated)"""
    linear_bwd_weight(a, h, dw2)
    colsum(a, db2)
    linear_bwd_weight(dh, p, dw1)
    colsum(dh, db1)


# ---- dense / rnn / misc -----------------------------------------------------------------------------------
DENSE_TF32 = True  # dense layers on wgmma tf32 (the reference's cuDNN-RNN precision); False -> fp32 SIMT


def _tf32_ok(a, a_ms, a_ks, b, b_ks, b_ns, m, n, k):
    return (a_ks == 1 and b_ks == 1 and a_ms % 4 == 0 and b_ns % 4 == 0 and a.data_ptr() % 16 == 0
            and b.data_ptr() % 16 == 0 and k % 4 == 0 and n % 4 == 0)


_scratch = {}


def _scratch_f32(tag, shape, device):
    # keyed by the CURRENT STREAM too: weight-gradient GEMMs run on a side stream while the main stream may stage
    # another transpose of the same shape (two streams must never share a staging buffer)
    key = (tag, tuple(shape), device, torch.cuda.current_stream(device).cuda_stream)
    t = _scratch.get(key)
    if t is None:
        t = torch.empty(*shape, device=device)
        _scratch[key] = t
    return t


def transpose_f32(src, dst):
    """dst[c, r] = src[r, c] for 2-D fp32 tensors (row strides honoured)"""
    rows, cols = src.shape
    call("hb200_transpose_f32", ptr(src), src.stride(0), ptr(dst), dst.stride(0), rows, cols)


def sgemm(a, a_ms, a_ks, b, b_ks, b_ns, c, ldc, m, n, k, bias=None, alpha=1.0, accumulate=False, relu=False,
          tf32=False):
    if tf32 and DENSE_TF32 and alpha == 1.0 and _tf32_ok(a, a_ms, a_ks, b, b_ks, b_ns, m, n, k):
        call("hb200_tgemm", ptr(a), int(a_ms), int(a_ks), ptr(b), int(b_ks), int(b_ns), ptr(c), int(ldc), ptr(bias),
             m, n, k, int(bool(accumulate)), int(bool(relu)))
        return
    call("hb200_sgemm", ptr(a), int(a_ms), int(a_ks), ptr(b), int(b_ks), int(b_ns), ptr(c), int(ldc), ptr(bias),
         m, n, k, float(alpha), int(bool(accumulate)), int(bool(relu)))


def linear_fwd(x, w, bias, out, relu=False, ldc=None, tf32=False):
    """out[M,N] = x[M,K] @ w[N,K]^T + bias"""
    M, K = x.shape
    N = w.shape[0]
    sgemm(x, x.stride(0), 1, w, 1, w.stride(0), out, ldc if ldc is not None else out.stride(0), M, N, K,
          bias=bias, relu=relu, tf32=tf32)


def linear_bwd_input(dy, w, dx, ld_dy=None, accumulate=False, tf32=False):
    """dx[M,K] = dy[M,N] @ w[N,K]"""
    M, N = dy.shape
    K = w.shape[1]
    if tf32 and DENSE_TF32 and N % 4 == 0 and K % 4 == 0 and dy.stride(0) % 4 == 0:
        wt = _scratch_f32("wt", (K, N), w.device)       # W^T so that both operands are K-major
        transpose_f32(w, wt)
        sgemm(dy, dy.stride(0), 1, wt, 1, wt.stride(0), dx, dx.stride(0), M, K, N, accumulate=accumulate, tf32=True)
        return
    sgemm(dy, ld_dy if ld_dy is not None else dy.stride(0), 1, w, w.stride(0), 1, dx, dx.stride(0), M, K, N,
          accumulate=accumulate)


def linear_bwd_weight(dy, x, dw, accumulate=False, tf32=False):
    """dw[N,K] = dy[M,N]^T @ x[M,K]"""
    M, N = dy.shape
    K = x.shape[1]
    if tf32 and DENSE_TF32 and M % 4 == 0 and K % 4 == 0:
        dyt = _scratch_f32("dyt", (N, M), dy.device)    # dy^T [N, frames], x^T [K, frames]: K-major operands
        xt = _scratch_f32("xt", (K, M), x.device)
        transpose_f32(dy, dyt)
        transpose_f32(x, xt)
        sgemm(dyt, M, 1, xt, 1, M, dw, dw.stride(0), N, K, M, accumulate=accumulate, tf32=True)
        return
    sgemm(dy, 1, dy.stride(0), x, x.stride(0), 1, dw, dw.stride(0), N, K, M, accumulate=accumulate)


def f16_to_bf16(x, out):
    call("hb200_f16_to_bf16", ptr(x), ptr(out), x.numel())


def bf16_to_f32(x, out):
    call("hb200_bf16_to_f32", ptr(x), ptr(out), x.numel())


def f32_to_bf16(x, out):
    call("hb200_f32_to_bf16", ptr(x), ptr(out), x.numel())


def lstm_step_fwd(xproj, w_hh, masks, h_prev, c_prev, h, c, gates_out, n, hidden, b_hh=None):
    call("hb200_lstm_step_fwd", ptr(xproj), ptr(w_hh), ptr(b_hh), ptr(masks), ptr(h_prev), h_prev.stride(0), ptr(c_prev),
         c_prev.stride(0), ptr(h), ptr(c), ptr(gates_out), n, hidden)


def lstm_step_bwd(dh_out, dh_rec, dc_rec, gates, c, c_prev, w_hh, masks, dgates, dh_prev, dc_prev, n, hidden):
    call("hb200_lstm_step_bwd", ptr(dh_out), ptr(dh_rec), ptr(dc_rec), ptr(gates), ptr(c), ptr(c_prev),
         c_prev.stride(0), ptr(w_hh), ptr(masks), ptr(dgates), ptr(dh_prev), ptr(dc_prev), n, hidden)


def lstm_seq_fwd(xproj, w_hh, b_hh, masks, h0, c0, hs, cs, gates, T, n, hidden, workspace):
    call("hb200_lstm_seq_fwd", ptr(xproj), ptr(w_hh), ptr(b_hh), ptr(masks), ptr(h0), h0.stride(0), ptr(c0),
         c0.stride(0), ptr(hs), ptr(cs), ptr(gates), T, n, hidden, ptr(workspace))


def lstm_seq_bwd(dh_out, gates, cs, c0, w_hh, masks, dgates, T, n, hidden, workspace):
    call("hb200_lstm_seq_bwd", ptr(dh_out), ptr(gates), ptr(cs), ptr(c0), c0.stride(0), ptr(w_hh), ptr(masks),
         ptr(dgates), T, n, hidden, ptr(workspace))


def lstm_seq_bwd_chunk(dh_out, gates, cs, c0, w_hh, masks, dgates, T, n, hidden, workspace, carry, carry_in, carry_out):
    """one time chunk of the backward recurrence; carry f32 [2, n, H] links it to its neighbours (see hb200.h)"""
    call("hb200_lstm_seq_bwd_chunk", ptr(dh_out), ptr(gates), ptr(cs), ptr(c0), c0.stride(0), ptr(w_hh), ptr(masks),
         ptr(dgates), T, n, hidden, ptr(workspace), ptr(carry), int(bool(carry_in)), int(bool(carry_out)))


def gru_seq_fwd(xproj, w_hh, b_hh, masks, h0, hs, saved, T, n, hidden, workspace):
    call("hb200_gru_seq_fwd", ptr(xproj), ptr(w_hh), ptr(b_hh), ptr(masks), ptr(h0), h0.stride(0), ptr(hs), ptr(saved),
         T, n, hidden, ptr(workspace))


def gru_seq_bwd(dh_out, saved, hs, h0, w_hh, masks, dgx, dgh, T, n, hidden, workspace):
    call("hb200_gru_seq_bwd", ptr(dh_out), ptr(saved), ptr(hs), ptr(h0), h0.stride(0), ptr(w_hh), ptr(masks), ptr(dgx),
         ptr(dgh), T, n, hidden, ptr(workspace))


def rnn_shift_mask(h_seq, h0, masks, h_in, T, n, hidden):
    call("hb200_rnn_shift_mask", ptr(h_seq), ptr(h0), h0.stride(0), ptr(masks), ptr(h_in), T, n, hidden)


def colsum(x, out, accumulate=False, n_cols=None):
    M = x.shape[0]
    N = x.shape[1] if n_cols is None else n_cols
    call("hb200_colsum", ptr(x), x.stride(0), ptr(out), M, N, int(bool(accumulate)))


def relu_bwd(d, y, cols):
    call("hb200_relu_bwd", ptr(d), ptr(y), d.stride(0), y.stride(0), d.shape[0], cols)


def gather_rows(src, frame_rows, out):
    """out[f] = src[frame_rows[f]] for f32 src [R, F] and out [B, F] (both contiguous), frame_rows int32 [B]"""
    _chk(src, torch.float32, "gather_rows src")
    _chk(out, torch.float32, "gather_rows out")
    _chk(frame_rows, torch.int32, "gather_rows frame_rows")
    if src.dim() != 2 or out.dim() != 2 or out.shape != (frame_rows.numel(), src.shape[1]):
        raise _lib.Hb200Error(f"gather_rows: src {tuple(src.shape)}, rows {frame_rows.numel()}, out {tuple(out.shape)}")
    call("hb200_gather_rows", ptr(src), ptr(frame_rows), ptr(out), out.shape[0], out.shape[1])


def f32_chw_to_bf16_hwc(x, out, batch, hw, channels):
    call("hb200_f32_chw_to_bf16_hwc", ptr(x), ptr(out), batch, hw, channels)


def heads_fwd(features, w_act, b_act, w_val, b_val, logits, values):
    B, H = features.shape
    call("hb200_heads_fwd", ptr(features), ptr(w_act), ptr(b_act), ptr(w_val), ptr(b_val), B, H, w_act.shape[0],
         ptr(logits), ptr(values))


def heads_act(features, w_act, b_act, w_val, b_val, uniform, log_probs, values, actions, action_log_probs):
    """uniform: f32 [B] in [0,1) for a draw, or None for the mode."""
    B, H = features.shape
    assert actions.dtype == torch.int64
    call("hb200_heads_act", ptr(features), ptr(w_act), ptr(b_act), ptr(w_val), ptr(b_val),
         ptr(uniform), B, H, w_act.shape[0], ptr(log_probs), ptr(values), ptr(actions),
         ptr(action_log_probs))


def embed_fwd(goal, prev_actions, masks, frame_rows, w_tgt, b_tgt, emb, out, col0):
    call("hb200_embed_fwd", ptr(goal), ptr(prev_actions), ptr(as_u8(masks)), ptr(frame_rows), ptr(w_tgt),
         ptr(b_tgt), ptr(emb), ptr(out), out.stride(0), col0, frame_rows.numel())


def embed_bwd(goal, prev_actions, masks, frame_rows, d_out, col0, d_w_tgt, d_b_tgt, d_emb):
    call("hb200_embed_bwd", ptr(goal), ptr(prev_actions), ptr(as_u8(masks)), ptr(frame_rows), ptr(d_out),
         d_out.stride(0), col0, frame_rows.numel(), d_emb.shape[0], ptr(d_w_tgt), ptr(d_b_tgt), ptr(d_emb))


# ---- generic 1-D sensors / embeddings / visual prep (any sensor set of PointNavResNetNet) ----------------
T_IDENTITY, T_POLAR2, T_POLAR3, T_COSSIN = 0, 1, 2, 3


def sensor_linear_fwd(x, frame_rows, transform, w, b, out, col0, out_dim):
    """x f32 [rows, in_dim] observation buffer; out f32 [B, ld]: columns [col0, col0 + out_dim) (see hb200.h)"""
    call("hb200_sensor_linear_fwd", ptr(x), x.shape[-1], ptr(frame_rows), frame_rows.numel(), int(transform), ptr(w),
         ptr(b), ptr(out), out.stride(0), int(col0), int(out_dim))


def sensor_linear_bwd(x, frame_rows, transform, d_out, col0, out_dim, d_w, d_b):
    call("hb200_sensor_linear_bwd", ptr(x), x.shape[-1], ptr(frame_rows), frame_rows.numel(), int(transform),
         ptr(d_out), d_out.stride(0), int(col0), int(out_dim), ptr(d_w), ptr(d_b))


def index_embed_fwd(idx, frame_rows, masks, table, out, col0, batch):
    call("hb200_index_embed_fwd", ptr(idx), ptr(frame_rows), ptr(as_u8(masks) if masks is not None else None), int(batch),
         table.shape[0], ptr(table), table.shape[1], ptr(out), out.stride(0), int(col0))


def index_embed_bwd(idx, frame_rows, masks, d_out, col0, d_table, batch):
    call("hb200_index_embed_bwd", ptr(idx), ptr(frame_rows), ptr(as_u8(masks) if masks is not None else None), int(batch),
         d_table.shape[0], d_table.shape[1], ptr(d_out), d_out.stride(0), int(col0), ptr(d_table))


_PREP_DTYPE = {torch.uint8: 0, torch.float32: 1, torch.int32: 2}


def prep_generic(sources, frame_rows, H, W, scale_shift=None, out=None, out_bf16=None, stats_acc=None):
    """sources: list of (tensor [rows, H, W, C] u8 / f32 / i32, scale).  Either `stats_acc` (statistics pass) or `out`."""
    n = len(sources)
    ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t, _ in sources])
    dts = (ctypes.c_int * n)(*[_PREP_DTYPE[t.dtype] for t, _ in sources])
    chs = (ctypes.c_int * n)(*[t.shape[-1] for t, _ in sources])
    scs = (ctypes.c_float * n)(*[float(s) for _, s in sources])
    call("hb200_prep_generic", ctypes.addressof(ptrs), ctypes.addressof(dts), ctypes.addressof(chs),
         ctypes.addressof(scs), n, ptr(frame_rows), frame_rows.numel(), int(H), int(W), ptr(scale_shift), ptr(out),
         ptr(out_bf16), ptr(stats_acc))


# ---- observation transforms -----------------------------------------------------------------------------
OBS_AREA, OBS_NEAREST, OBS_COPY = 0, 1, 2
OBS_MAX_KEYS = 8


def obs_resample(keys):
    """Resample and window NHWC image batches, every key in one launch (ResizeShortestEdge / CenterCropper).

    keys: list of (src [B, H, W, C], dst [B, h, w, C], mode, (Hr, Wr), (y0, x0)).  dst receives rows y0 .. y0+h-1 and
    columns x0 .. x0+w-1 of src resampled to Hr x Wr: OBS_AREA / OBS_NEAREST as F.interpolate(src.float(), (Hr, Wr),
    mode).to(src.dtype) computes them on the CPU, bit for bit (u8, f32, i32); OBS_COPY needs (Hr, Wr) = (H, W) and
    copies the window's bits for any dtype.  Every tensor must be a contiguous CUDA tensor; dst may be a view into a
    larger buffer (e.g. one time slot of the rollout storage) as long as it is contiguous."""
    if not 1 <= len(keys) <= OBS_MAX_KEYS:
        raise _lib.Hb200Error(f"obs_resample: {len(keys)} keys (1..{OBS_MAX_KEYS} per launch)")
    srcs, dsts, desc, batch = [], [], [], None
    for i, (src, dst, mode, (hr, wr), (y0, x0)) in enumerate(keys):
        what = f"obs_resample key {i}"
        if src.dim() != 4 or dst.dim() != 4:
            raise _lib.Hb200Error(f"{what}: expected 4-D NHWC tensors, got {tuple(src.shape)} -> {tuple(dst.shape)}")
        if mode not in (OBS_AREA, OBS_NEAREST, OBS_COPY):
            raise _lib.Hb200Error(f"{what}: unknown mode {mode}")
        if mode == OBS_COPY:
            src, dst = src.view(torch.uint8), dst.view(torch.uint8)  # bits of any dtype, as u8 channels
        elif src.dtype not in _PREP_DTYPE:
            raise _lib.Hb200Error(f"{what}: dtype {src.dtype} (uint8, float32 or int32)")
        _chk(src, src.dtype, f"{what} src")
        _chk(dst, src.dtype, f"{what} dst")
        if src.device != dst.device:
            raise _lib.Hb200Error(f"{what}: src on {src.device}, dst on {dst.device}")
        B, H, W, C = src.shape
        _, h, w, c = dst.shape
        batch = B if batch is None else batch
        if B != batch or dst.shape[0] != B or c != C:
            raise _lib.Hb200Error(f"{what}: shapes {tuple(src.shape)} -> {tuple(dst.shape)} (batch {batch})")
        if mode == OBS_COPY and (hr, wr) != (H, W):
            raise _lib.Hb200Error(f"{what}: copy keeps the size ({H}, {W}), got ({hr}, {wr})")
        if not (hr >= 1 and wr >= 1 and 0 <= y0 and 0 <= x0 and y0 + h <= hr and x0 + w <= wr):
            raise _lib.Hb200Error(f"{what}: window ({y0}, {x0}, {h}, {w}) outside the resampled {hr}x{wr} image")
        if B == 0 or h == 0 or w == 0:
            raise _lib.Hb200Error(f"{what}: empty tensor {tuple(dst.shape)}")
        srcs.append(src.data_ptr())
        dsts.append(dst.data_ptr())
        desc += [_PREP_DTYPE[src.dtype], mode, H, W, C, int(hr), int(wr), int(y0), int(x0), h, w]
    n = len(keys)
    src_a = (ctypes.c_void_p * n)(*srcs)
    dst_a = (ctypes.c_void_p * n)(*dsts)
    desc_a = (ctypes.c_int32 * len(desc))(*desc)
    call("hb200_obs_resample", ctypes.addressof(src_a), ctypes.addressof(dst_a), ctypes.addressof(desc_a), n, batch)


# ---- experimental probes (not on the product path) ------------------------------------------------------
def tma_halo_probe(x, out, b, oh0, ow0, halo_h, halo_w, pad):
    """x bf16 [B,H,W,C] -> out bf16 [C/8, halo_h, halo_w, 8]: one tile's input halo loaded by TMA (see hb200.h)."""
    B, H, W, C = x.shape
    call("hb200_tma_halo_probe", ptr(x), ptr(out), B, H, W, C, int(b), int(oh0), int(ow0), int(halo_h), int(halo_w), int(pad))
