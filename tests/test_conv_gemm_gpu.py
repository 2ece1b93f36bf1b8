"""wgmma convolution GEMM vs a plain torch fp32 convolution of the same fp16-rounded operands."""
import ctypes

import pytest
import torch

from crazyara_b200 import check, lib


def _run_conv(boards, cin, n_out, ksize, relu, use_res, bn, f32_out=False, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    dev = "cuda"
    boards_cap = boards + (boards & 1)
    boards_cap = max(boards_cap, 2)
    act = (torch.randn(boards_cap, 8, 8, cin, generator=g) * 0.5).half()
    taps = ksize * ksize
    cw = (cin + 63) // 64 * 64
    w = (torch.randn(n_out, cin, ksize, ksize, generator=g) / (cin * taps) ** 0.5).half()
    bias = torch.randn(n_out, generator=g) * 0.1
    ldo = (n_out + 31) // 32 * 32
    if bn == 0:
        bn = lib().ara_debug_choose_bn(boards, n_out)
    w_rows = (n_out + bn - 1) // bn * bn
    # kernel weight layout: [w_rows, taps * cw], k = tap * cw + c, tap = ky * ksize + kx
    wk = torch.zeros(w_rows, taps, cw, dtype=torch.half)
    wk[:n_out, :, :cin] = w.permute(0, 2, 3, 1).reshape(n_out, taps, cin)
    wk = wk.reshape(w_rows, taps * cw).contiguous()
    bias_p = torch.zeros(ldo)
    bias_p[:n_out] = bias
    res = (torch.randn(boards * 64, ldo, generator=g) * 0.5).half() if use_res else None

    act_d, wk_d, bias_d = act.to(dev), wk.to(dev), bias_p.to(dev)
    res_d = res.to(dev) if use_res else None
    out_h = torch.full((boards * 64, ldo), float("nan"), dtype=torch.half, device=dev)
    out_f = torch.full((boards * 64, ldo), float("nan"), dtype=torch.float32, device=dev) if f32_out else None
    rc = lib().ara_debug_conv(
        ctypes.c_void_p(act_d.data_ptr()), boards_cap, boards, cin, ctypes.c_void_p(wk_d.data_ptr()), w_rows, n_out,
        ksize, ctypes.c_void_p(bias_d.data_ptr()), int(relu),
        ctypes.c_void_p(res_d.data_ptr() if use_res else 0), ldo,
        ctypes.c_void_p(0 if f32_out else out_h.data_ptr()), ctypes.c_void_p(out_f.data_ptr() if f32_out else 0),
        ldo, bn, ctypes.c_void_p(0))
    check(rc)
    torch.cuda.synchronize()
    # reference: fp32 conv on the same fp16-rounded operands
    x = act[:boards].float().permute(0, 3, 1, 2).to(dev)
    ref = torch.nn.functional.conv2d(x, w.float().to(dev), bias.to(dev), padding=ksize // 2)
    if relu:
        ref = torch.relu(ref)
    ref = ref.permute(0, 2, 3, 1).reshape(boards * 64, n_out)
    if use_res:
        ref = ref + res_d[:, :n_out].float()
    got = (out_f if f32_out else out_h.float())[:, :n_out]
    pad = (out_f if f32_out else out_h.float())[:, n_out:]
    return got, ref, pad


CASES = [
    # boards, cin, n_out, ksize, relu, res, bn
    (2, 256, 256, 1, True, False, 64),
    (2, 64, 256, 3, True, False, 64),
    (8, 256, 128, 1, True, False, 128),
    (8, 256, 896, 1, True, False, 128),
    (8, 896, 256, 1, False, True, 64),
    (64, 256, 256, 3, True, False, 128),
    (64, 256, 256, 3, True, False, 256),
    (64, 224, 256, 1, False, True, 0),
    (64, 256, 224, 1, True, False, 0),
    (1, 64, 256, 3, True, False, 0),
    (5, 256, 352, 1, True, False, 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("boards,cin,n_out,ksize,relu,res,bn", CASES)
def test_conv_gemm_matches_torch(boards, cin, n_out, ksize, relu, res, bn):
    got, ref, pad = _run_conv(boards, cin, n_out, ksize, relu, res, bn)
    assert torch.isfinite(got).all()
    err = (got - ref).abs().max().item()
    # fp16 output rounding: |x| <= ~8 -> half ulp 4e-3
    assert err < 1.5e-2, f"max abs err {err}"
    if pad.numel():
        assert (pad == 0).all()


@pytest.mark.gpu
def test_conv_gemm_policy_logits_fp32():
    got, ref, pad = _run_conv(64, 256, 81, 3, False, False, 0, f32_out=True)
    err = (got - ref).abs().max().item()
    assert err < 2e-3, f"max abs err {err}"
    assert (pad == 0).all()
