"""Kernel-level parity (-m gpu): every CUDA op of libvd3d_b200 against the fp32 CPU oracle ops, through the C ABI."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import torch_port as tp

pytestmark = pytest.mark.gpu


def _E():
    from visualdet3d_b200 import engine
    return engine


def nhwc(x_nchw):
    return x_nchw.permute(0, 2, 3, 1).contiguous()


CONV_CASES = [
    # B, Cin, H, W, Cout, k, stride, pad, dil, bias, res, relu
    (2, 3, 33, 47, 64, 7, 2, 3, 1, False, False, True),      # stem (scalar gather path)
    (2, 4, 33, 47, 64, 7, 2, 3, 1, False, False, True),      # stem, padded to 4 channels
    (1, 64, 24, 40, 64, 3, 1, 1, 1, False, True, True),
    (2, 64, 24, 40, 128, 3, 2, 1, 1, False, False, True),
    (2, 64, 24, 40, 128, 1, 2, 0, 1, False, False, False),   # downsample
    (1, 24, 17, 23, 24, 3, 1, 1, 1, False, False, True),     # K tail (216 = 13.5 chunks)
    (1, 72, 12, 20, 72, 3, 1, 1, 1, True, True, True),
    (1, 256, 6, 20, 8, 1, 1, 0, 1, True, False, True),       # cost-volume down-sample (Cout = 8)
    (1, 256, 6, 20, 144, 3, 1, 1, 1, True, False, False),
    (1, 128, 9, 11, 256, 3, 1, 2, 2, True, False, True),     # dilation 2
    (1, 1408, 6, 20, 256, 3, 1, 1, 1, True, False, True),
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv2d_vs_torch(case):
    E = _E()
    B, Cin, H, W, Cout, k, s, p, d, has_b, has_r, relu = case
    g = torch.Generator().manual_seed(sum(case[:6]))
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g) if has_b else None
    ref = F.conv2d(x, w, b, stride=s, padding=p, dilation=d)
    r = torch.randn(ref.shape, generator=g) if has_r else None
    if r is not None:
        ref = ref + r
    if relu:
        ref = F.relu(ref)
    layer = E.ConvLayer(w, b, None, stride=s, pad=p, dil=d, relu=relu, device="cuda", engine="simt")
    xa = E.Act(nhwc(x).cuda())
    Ho, Wo = layer.out_hw(H, W)
    # write into a channel slice of a wider buffer to exercise pitch / offset handling
    out = E.Act(torch.full((B, Ho, Wo, Cout + 8), 7.0, device="cuda"), 4, Cout)
    ra = E.Act(nhwc(r).cuda()) if r is not None else None
    layer(xa, out, res=ra)
    got = out.to_nchw().cpu()
    assert float(out.t[..., :4].min()) == 7.0 and float(out.t[..., 4 + Cout:].min()) == 7.0   # neighbours untouched
    np.testing.assert_allclose(got.numpy(), ref.numpy(), rtol=1e-4, atol=2e-5)


def test_conv_bn_folding_matches_conv_then_bn():
    E = _E()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 32, 10, 12, generator=g)
    w = torch.randn(48, 32, 3, 3, generator=g) * 0.1
    bn = dict(weight=torch.rand(48, generator=g) + 0.5, bias=torch.randn(48, generator=g) * 0.1,
              running_mean=torch.randn(48, generator=g) * 0.1, running_var=torch.rand(48, generator=g) + 0.5)
    ref = F.relu(F.batch_norm(F.conv2d(x, w, None, padding=1), bn["running_mean"], bn["running_var"], bn["weight"], bn["bias"], False, 0.0, 1e-5))
    layer = E.ConvLayer(w, None, bn, pad=1, relu=True, device="cuda", engine="simt")
    out = layer(E.Act(nhwc(x).cuda()), E.Act(torch.empty(2, 10, 12, 48, device="cuda")))
    np.testing.assert_allclose(out.to_nchw().cpu().numpy(), ref.numpy(), rtol=1e-4, atol=2e-5)


@pytest.mark.parametrize("shape", [(2, 64, 5, 80), (1, 128, 3, 40), (1, 64, 4, 200), (2, 32, 3, 50), (1, 64, 2, 20), (1, 128, 2, 7)])
def test_psm_cosine_vs_oracle(shape):
    """PSMCosine (R/lib/PSM_cost_volume.py:76-91): tiled kernel (C = 64/128, D = 24), generic kernel, ragged widths,
    W < D (planes beyond the width stay zero)."""
    E = _E()
    B, C, H, W = shape
    g = torch.Generator().manual_seed(C + W)
    L, R = torch.randn(B, C, H, W, generator=g), torch.randn(B, C, H, W, generator=g)
    ref = tp.psm_cosine(L, R, 96, 4)
    out = E.Act(torch.full((B, H, W, 32), 3.0, device="cuda"), 4, 24)
    E.psm_cosine(E.Act(nhwc(L).cuda()), E.Act(nhwc(R).cuda()), 24, out)
    np.testing.assert_allclose(out.to_nchw().cpu().numpy(), ref.numpy(), rtol=1e-5, atol=2e-6)
    assert float(out.t[..., :4].min()) == 3.0 and float(out.t[..., 28:].min()) == 3.0
    # exact zeros where w < i
    got = out.to_nchw().cpu()
    for i in range(1, min(24, W)):
        assert float(got[:, i, :, :i].abs().max()) == 0.0
    # NCHW op-level mirror
    from visualdet3d_b200._lib import call
    o2 = torch.empty(B, 24, H, W, device="cuda")
    Lc, Rc = L.cuda(), R.cuda()
    call("vd3d_psm_cosine_nchw", Lc.data_ptr(), Rc.data_ptr(), B, C, H, W, 24, o2.data_ptr(), None)
    np.testing.assert_allclose(o2.cpu().numpy(), ref.numpy(), rtol=1e-5, atol=2e-6)


def test_psm_cosine_linearity_full_size():
    """Size-independent property at the BASELINE shape (B=8, 64ch, 96x320): cost(L, a*R1 + R2) = a*cost(L,R1) + cost(L,R2)."""
    E = _E()
    B, C, H, W = 8, 64, 96, 320
    g = torch.Generator(device="cuda").manual_seed(0)
    L = torch.randn(B, H, W, C, device="cuda", generator=g)
    R1 = torch.randn(B, H, W, C, device="cuda", generator=g)
    R2 = torch.randn(B, H, W, C, device="cuda", generator=g)
    outs = []
    for Rr in (R1, R2, 0.5 * R1 + R2):
        o = E.Act(torch.empty(B, H, W, 24, device="cuda"))
        E.psm_cosine(E.Act(L), E.Act(Rr.contiguous()), 24, o)
        outs.append(o.t)
    assert float((outs[2] - (0.5 * outs[0] + outs[1])).abs().max()) < 1e-5
    assert float(outs[0][:, :, 0, 1:].abs().max()) == 0.0        # w = 0: only disparity 0 is defined


def test_concat_volume_conv3d_vs_oracle():
    E = _E()
    from visualdet3d_b200._lib import call
    g = torch.Generator().manual_seed(9)
    B, Fc, H, W, D = 2, 8, 6, 20, 12
    lf, rf = torch.rand(B, Fc, H, W, generator=g), torch.rand(B, Fc, H, W, generator=g)
    w1, b1 = torch.randn(8, 16, 3, 3, 3, generator=g) * 0.1, torch.randn(8, generator=g) * 0.1
    w2, b2 = torch.randn(8, 8, 3, 3, 3, generator=g) * 0.1, torch.randn(8, generator=g) * 0.1
    vol = tp.concat_volume(lf, rf, D)
    ref = F.relu(F.conv3d(F.relu(F.conv3d(vol, w1, b1, padding=1)), w2, b2, padding=1)).reshape(B, -1, H, W)
    pk = lambda w: w.permute(2, 3, 4, 1, 0).reshape(27, w.shape[1], w.shape[0]).contiguous().cuda()
    mid = torch.empty(B, D, H, W, Fc, device="cuda")
    out = E.Act(torch.zeros(B, H, W, 100, device="cuda"), 4, 96)
    keep = [nhwc(lf).cuda(), nhwc(rf).cuda(), pk(w1), b1.cuda(), pk(w2), b2.cuda()]   # keep the device buffers alive
    call("vd3d_concat_volume_conv3d", keep[0].data_ptr(), keep[1].data_ptr(), B, H, W, Fc, D,
         keep[2].data_ptr(), keep[3].data_ptr(), keep[4].data_ptr(), keep[5].data_ptr(), mid.data_ptr(),
         out.ptr, out.cs, out.co, None)
    np.testing.assert_allclose(out.to_nchw().cpu().numpy(), ref.numpy(), rtol=1e-4, atol=1e-5)


# ----------------------------------------------------------------------------------------------------------------
# wgmma conv engine
# ----------------------------------------------------------------------------------------------------------------
def _trunc13(t):
    return (t.contiguous().view(torch.int32) & -8192).view(torch.float32)


def test_tc_mma_reads_top_19_bits_only():
    """Hardware probe the 3xTF32 split relies on: kind::tf32 must use exactly x & 0xFFFFE000 of a 32-bit operand.
    1x1 conv with power-of-two weights (products exact) in single-pass mode == conv(trunc13(x), w) bit for bit."""
    E = _E()
    g = torch.Generator().manual_seed(3)
    B, C, H, W, Co = 1, 32, 8, 16, 16
    x = torch.randn(B, C, H, W, generator=g)
    w = torch.zeros(Co, C, 1, 1)
    for o in range(Co):
        w[o, (o * 5) % C, 0, 0] = 2.0 ** (o % 5 - 2)
    layer = E.ConvLayer(w, None, None, relu=False, device="cuda", engine="tc1")
    assert layer.engine == "tc1"
    out = layer(E.Act(nhwc(x).cuda()), E.Act(torch.empty(B, H, W, Co, device="cuda")))
    got = out.to_nchw().cpu()
    exp_trunc = F.conv2d(_trunc13(x), w)
    exp_plain = F.conv2d(x, w)
    d_trunc = float((got - exp_trunc).abs().max())
    d_plain = float((got - exp_plain).abs().max())
    print("tf32 operand probe: |got - trunc| =", d_trunc, " |got - fp32| =", d_plain)
    assert d_trunc == 0.0, "tensor core does not truncate fp32 operands to their top 19 bits"


TC_CASES = [
    # B, Cin, H, W, Cout, k, pad, dil, bias, res, relu
    (1, 32, 8, 16, 16, 1, 0, 1, False, False, False),
    (2, 64, 24, 40, 64, 3, 1, 1, False, True, True),
    (1, 64, 18, 80, 64, 3, 1, 1, True, False, True),       # H not a multiple of the 8-row tile
    (1, 96, 12, 20, 96, 3, 1, 1, False, False, True),      # BN = 96
    (1, 256, 6, 20, 144, 3, 1, 1, True, False, False),     # BN = 144 (single N tile)
    (1, 128, 9, 11, 256, 3, 2, 2, True, True, True),       # dilation 2, ragged tile
    (1, 288, 6, 20, 288, 3, 1, 1, False, True, True),
    (2, 1408, 6, 20, 256, 3, 1, 1, True, False, True),     # long K (396 k-blocks)
    (1, 256, 6, 20, 576, 3, 1, 1, True, False, False),
]


@pytest.mark.parametrize("case", TC_CASES)
def test_conv2d_tc_3xtf32_vs_fp32(case):
    E = _E()
    B, Cin, H, W, Cout, k, p, d, has_b, has_r, relu = case
    g = torch.Generator().manual_seed(sum(case[:6]))
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g) if has_b else None
    ref64 = F.conv2d(x.double(), w.double(), b.double() if b is not None else None, padding=p, dilation=d)
    r = torch.randn(ref64.shape, generator=g) if has_r else None
    if r is not None:
        ref64 = ref64 + r.double()
    if relu:
        ref64 = F.relu(ref64)
    layer = E.ConvLayer(w, b, None, pad=p, dil=d, relu=relu, device="cuda", engine="tc")
    assert layer.engine == "tc"
    xa = E.split_lo(E.Act(nhwc(x).cuda(), 0, None, torch.zeros(B, H, W, Cin, device="cuda")))
    Ho, Wo = layer.out_hw(H, W)
    out = E.Act(torch.full((B, Ho, Wo, Cout + 8), 7.0, device="cuda"), 4, Cout, torch.full((B, Ho, Wo, Cout + 8), 7.0, device="cuda"))
    layer(xa, out, res=E.Act(nhwc(r).cuda()) if r is not None else None)
    got = out.to_nchw().cpu()
    err = float((got.double() - ref64).abs().max())
    # same conv on the exact-fp32 SIMT engine, for scale
    simt = E.ConvLayer(w, b, None, pad=p, dil=d, relu=relu, device="cuda", engine="simt")
    o2 = simt(E.Act(nhwc(x).cuda()), E.Act(torch.empty(B, Ho, Wo, Cout, device="cuda")), res=E.Act(nhwc(r).cuda()) if r is not None else None)
    err_simt = float((o2.to_nchw().cpu().double() - ref64).abs().max())
    print(case, "max|err| vs fp64: 3xTF32", err, " fp32-SIMT", err_simt)
    assert err < 2e-5, err
    assert float(out.t[..., :4].min()) == 7.0 and float(out.t[..., 4 + Cout:].min()) == 7.0
    # lo companion written by the epilogue
    got_lo = out.lo[..., 4:4 + Cout].cpu()
    val = out.t[..., 4:4 + Cout].cpu()
    assert torch.equal(got_lo, val - _trunc13(val))


@pytest.mark.parametrize("case", TC_CASES)
def test_conv2d_tc16_fp16split_vs_fp64(case):
    """fp16-split tensor-core conv (3 kind::f16 MMAs on (hi, lo) fp16 planes, 22 significant bits): same accuracy bar as the
    3xTF32 form, checked against an fp64 convolution; also checks the fp16 planes the epilogue writes for the next layer."""
    E = _E()
    B, Cin, H, W, Cout, k, p, d, has_b, has_r, relu = case
    g = torch.Generator().manual_seed(sum(case[:6]) + 1)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g) if has_b else None
    ref64 = F.conv2d(x.double(), w.double(), b.double() if b is not None else None, padding=p, dilation=d)
    r = torch.randn(ref64.shape, generator=g) if has_r else None
    if r is not None:
        ref64 = ref64 + r.double()
    if relu:
        ref64 = F.relu(ref64)
    layer = E.ConvLayer(w, b, None, pad=p, dil=d, relu=relu, device="cuda", engine="tc16")
    assert layer.engine == "tc16"
    xa = E.split_lo(E.Act(nhwc(x).cuda(), 0, None, torch.zeros(2, B, H, W, Cin, device="cuda", dtype=torch.float16)))
    Ho, Wo = layer.out_hw(H, W)
    out = E.Act(torch.full((B, Ho, Wo, Cout + 16), 7.0, device="cuda"), 8, Cout,
                torch.full((2, B, Ho, Wo, Cout + 16), 7.0, device="cuda", dtype=torch.float16))
    layer(xa, out, res=E.Act(nhwc(r).cuda()) if r is not None else None)
    got = out.to_nchw().cpu()
    err = float((got.double() - ref64).abs().max())
    print(case, "max|err| vs fp64: fp16-split", err)
    assert err < 2e-5, err
    assert float(out.t[..., :8].min()) == 7.0 and float(out.t[..., 8 + Cout:].min()) == 7.0
    val = out.t[..., 8:8 + Cout]
    hi = val.half()
    assert torch.equal(out.lo[0][..., 8:8 + Cout], hi)
    assert torch.equal(out.lo[1][..., 8:8 + Cout], (val - hi.float()).half())
    assert float(out.lo[..., :8].float().min()) == 7.0 and float(out.lo[..., 8 + Cout:].float().min()) == 7.0


def test_tc16_large_and_tiny_magnitudes():
    """weights are pre-scaled by a power of two so their fp16 lo parts stay normal; activations spanning 1e-3..1e3 keep
    a relative error of ~2^-21 against fp64."""
    E = _E()
    g = torch.Generator().manual_seed(5)
    for wscale, xscale in ((1e-3, 1.0), (30.0, 1.0), (1.0, 300.0), (1.0, 1e-2)):
        x = torch.randn(1, 64, 16, 24, generator=g) * xscale
        w = torch.randn(32, 64, 3, 3, generator=g) * wscale / 24.0
        ref64 = F.conv2d(x.double(), w.double(), padding=1)
        layer = E.ConvLayer(w, None, None, pad=1, relu=False, device="cuda", engine="tc16")
        xa = E.split_lo(E.Act(nhwc(x).cuda(), 0, None, torch.zeros(2, 1, 16, 24, 64, device="cuda", dtype=torch.float16)))
        out = layer(xa, E.Act(torch.empty(1, 16, 24, 32, device="cuda")))
        rel = float((out.to_nchw().cpu().double() - ref64).abs().max() / ref64.abs().max())
        print("wscale", wscale, "xscale", xscale, "rel err", rel)
        assert rel < 4e-6, (wscale, xscale, rel)


def test_fp16_range_guard():
    """The fp16-split engine keeps activations UNSCALED as fp16 (hi, lo) planes: |v| >= 65520 cannot be represented (hi = inf).  Every
    kernel that writes such planes raises a device flag instead of silently producing inf / NaN: the splitter, the conv epilogue
    (output planes), and -- end to end -- the detector (`Vd3dError` from `results()` and from the streamed pipeline's record block)."""
    E = _E()
    from visualdet3d_b200._lib import Vd3dError
    g = torch.Generator().manual_seed(7)
    assert not E.fp16_range_overflowed()
    planes = lambda *s: torch.zeros(2, *s, device="cuda", dtype=torch.float16)
    # (a) splitter: 65519 still rounds to the largest finite fp16, 65520 does not
    x = torch.randn(1, 64, 16, 24, generator=g)
    x[0, 3, 2, 5] = 65519.0
    E.split_lo(E.Act(nhwc(x).cuda(), 0, None, planes(1, 16, 24, 64)))
    assert not E.fp16_range_overflowed()
    x[0, 3, 2, 5] = -65520.0
    xa = E.split_lo(E.Act(nhwc(x).cuda(), 0, None, planes(1, 16, 24, 64)))
    assert E.fp16_range_overflowed() and not E.fp16_range_overflowed()           # reading clears it
    assert bool(torch.isinf(xa.lo[0].float()).any())
    # (b) conv epilogue: in-range inputs, an output beyond the range; without output planes nothing is flagged (fp32 output is exact)
    x = torch.randn(1, 64, 16, 24, generator=g) * 1000
    w = torch.randn(32, 64, 3, 3, generator=g)
    layer = E.ConvLayer(w, None, None, pad=1, relu=False, device="cuda", engine="tc16")
    xa = E.split_lo(E.Act(nhwc(x).cuda(), 0, None, planes(1, 16, 24, 64)))
    assert not E.fp16_range_overflowed()
    out32 = layer(xa, E.Act(torch.empty(1, 16, 24, 32, device="cuda")))
    assert float(out32.t.abs().max()) > 65520 and not E.fp16_range_overflowed()
    layer(xa, E.Act(torch.empty(1, 16, 24, 32, device="cuda"), 0, None, planes(1, 16, 24, 32)))
    assert E.fp16_range_overflowed()
    # (c) end to end: a frame scaled out of range makes the detector raise instead of returning detections; the next forward is clean
    from visualdet3d_b200 import synth
    from visualdet3d_b200.detectors import build_synthetic_stereo3d
    from visualdet3d_b200.pipeline import StreamedInference
    det, *_ = build_synthetic_stereo3d(seed=0)
    det = det.cuda().eval()
    left, right, P2, _ = synth.synth_stereo_inputs(1, 96, 320, seed=1)
    with torch.no_grad():
        with pytest.raises(Vd3dError, match="fp16 range"):
            det.forward_batch(left.cuda() * 1e6, right.cuda() * 1e6, P2.cuda())
        good = det.forward_batch(left.cuda(), right.cuda(), P2.cuda())
        assert len(good[0][0]) > 0
    pipe = StreamedInference(det, 1, 96, 320, kmax=64)
    t = pipe.submit((left * 1e6).pin_memory(), (right * 1e6).pin_memory(), P2.pin_memory())
    with pytest.raises(Vd3dError, match="fp16 range"):
        pipe.collect(t)
    t = pipe.submit(left.pin_memory(), right.pin_memory(), P2.pin_memory())
    got = pipe.collect(t)
    assert torch.equal(got[0][0], good[0][0].cpu())


TC16_EXTRA = [
    # B, Cin, H, W, Cout, k, pad, stride
    (2, 64, 24, 40, 128, 3, 1, 2),       # ResNet stage entry: 3x3 stride 2
    (1, 64, 17, 33, 128, 1, 0, 2),       # 1x1 stride-2 down-sample, odd sizes
    (1, 128, 20, 36, 256, 3, 1, 2),
    (1, 72, 12, 20, 72, 3, 1, 1),        # 72 channels: zero-filled up to the 64-channel k-block, Cout masked inside an 80-wide tile
    (1, 40, 16, 32, 40, 1, 0, 1),
    (1, 32, 15, 21, 64, 3, 1, 2),
]


@pytest.mark.parametrize("case", TC16_EXTRA)
def test_conv2d_tc16_strided_and_ragged_channels(case):
    """stride > 1 goes through the TMA traversal stride (every stride-th pixel lands densely in shared memory);
    channel counts that are not multiples of the 64-channel k-block / 16-column MMA granule are zero-filled / masked."""
    E = _E()
    B, Cin, H, W, Cout, k, p, s_ = case
    g = torch.Generator().manual_seed(sum(case))
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    ref64 = F.relu(F.conv2d(x.double(), w.double(), b.double(), padding=p, stride=s_))
    layer = E.ConvLayer(w, b, None, stride=s_, pad=p, relu=True, device="cuda", engine="tc16")
    assert layer.engine == "tc16"
    xa = E.split_lo(E.Act(nhwc(x).cuda(), 0, None, torch.zeros(2, B, H, W, Cin, device="cuda", dtype=torch.float16)))
    Ho, Wo = layer.out_hw(H, W)
    assert (Ho, Wo) == tuple(ref64.shape[2:])
    out = E.Act(torch.full((B, Ho, Wo, Cout + 8), 7.0, device="cuda"), 4, Cout,
                torch.full((2, B, Ho, Wo, Cout + 8), 7.0, device="cuda", dtype=torch.float16))
    layer(xa, out)
    err = float((out.to_nchw().cpu().double() - ref64).abs().max())
    print(case, "max|err| vs fp64", err)
    assert err < 2e-5, err
    assert float(out.t[..., :4].min()) == 7.0 and float(out.t[..., 4 + Cout:].min()) == 7.0
    assert float(out.lo[..., :4].float().min()) == 7.0 and float(out.lo[..., 4 + Cout:].float().min()) == 7.0


def test_conv2d_tc16_persistent_many_tiles():
    """more output tiles than SMs (every CTA loops several times, the TMA ring and the chunk promotion wrap across tiles),
    an odd number of M tiles (the second CTA of the last pair is dead) and several N tiles; checked against the exact-fp32
    SIMT engine of the same library."""
    E = _E()
    g = torch.Generator().manual_seed(11)
    # Cout = 608 -> three tiles of 208 columns, the last one ragged (192 valid); 1408 -> six tiles of 240 (last 208): the head shape
    for (B, Cin, H, W, Cout) in ((3, 64, 40, 112, 64), (1, 128, 24, 80, 384), (5, 64, 24, 48, 96), (3, 64, 24, 48, 608), (1, 64, 24, 80, 1408),
                                 (1, 64, 17, 23, 100)):
        x = torch.randn(B, H, W, Cin, generator=g)
        w = torch.randn(Cout, Cin, 3, 3, generator=g) / np.sqrt(Cin * 9)
        b = torch.randn(Cout, generator=g)
        r = torch.randn(B, H, W, Cout, generator=g)
        tc = E.ConvLayer(w, b, None, pad=1, relu=True, device="cuda", engine="tc16")
        simt = E.ConvLayer(w, b, None, pad=1, relu=True, device="cuda", engine="simt")
        xa = E.split_lo(E.Act(x.cuda(), 0, None, torch.zeros(2, B, H, W, Cin, device="cuda", dtype=torch.float16)))
        ra = E.Act(r.cuda())
        ref = simt(E.Act(xa.t), E.Act(torch.empty(B, H, W, Cout, device="cuda")), res=ra).t
        out = tc(xa, E.Act(torch.zeros(B, H, W, Cout, device="cuda"), 0, None, torch.zeros(2, B, H, W, Cout, device="cuda", dtype=torch.float16)), res=ra)
        err = float((out.t - ref).abs().max())
        print((B, Cin, H, W, Cout), "max|tc16 - simt|", err)
        assert err < 2e-5, err
        hi = out.t.half()
        assert torch.equal(out.lo[0], hi) and torch.equal(out.lo[1], (out.t - hi.float()).half())


def test_conv2d_tc16_tile_policies_are_bit_identical():
    """The tile policy depends on the problem size (tile width), so the same layer may run with different tiles at different batch
    sizes: every tile width must accumulate in the same order and give bit-identical results (batch invariance of the detectors rests
    on this)."""
    E = _E()
    g = torch.Generator().manual_seed(3)
    B, Cin, H, W, Cout = 2, 128, 24, 80, 384
    x = torch.randn(B, H, W, Cin, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / np.sqrt(Cin * 9)
    b = torch.randn(Cout, generator=g)
    layer = E.ConvLayer(w, b, None, pad=1, relu=True, device="cuda", engine="tc16")
    xa = E.split_lo(E.Act(x.cuda(), 0, None, torch.zeros(2, B, H, W, Cin, device="cuda", dtype=torch.float16)))
    outs = {}
    for bn in (0, 96, 128, 192):
        layer.bn_tile = bn
        outs[bn] = layer(xa, E.Act(torch.zeros(B, H, W, Cout, device="cuda"))).t.clone()
    ref = outs[0]
    for k, v in outs.items():
        assert torch.equal(v, ref), k


@pytest.mark.parametrize("win", ["32", "64"])
@pytest.mark.parametrize("shape", [(2, 3, 64, 96), (1, 3, 37, 53), (3, 3, 96, 320)])
def test_stem_tensor_core_vs_fp64(shape, win, monkeypatch):
    """conv1 7x7 stride 2 + BN + ReLU (R/backbones/resnet.py:120-122) through the row-window tensor-core path
    (image -> zero-padded fp16 row planes -> KHx1 conv over 64 virtual channels) against an fp64 convolution."""
    E = _E()
    monkeypatch.setenv("VD3D_STEM_WIN", win)          # 32: 8-pixel windows on 64-byte swizzle rows (default), 64: 16-pixel windows on 128-byte rows
    B, C, H, W = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(B, C, H, W, generator=g) * 2.0
    w = torch.randn(64, C, 7, 7, generator=g) / np.sqrt(C * 49)
    bn = dict(weight=torch.rand(64, generator=g) + 0.5, bias=torch.randn(64, generator=g) * 0.1,
              running_mean=torch.randn(64, generator=g) * 0.1, running_var=torch.rand(64, generator=g) + 0.5)
    ref64 = F.relu(F.batch_norm(F.conv2d(x.double(), w.double(), None, stride=2, padding=3), bn["running_mean"].double(), bn["running_var"].double(),
                                bn["weight"].double(), bn["bias"].double(), False, 0.0, 1e-5))
    layer = E.StemLayer(w, bn, stride=2, pad=3, relu=True, device="cuda")
    Ho, Wo = layer.out_hw(H, W)
    assert (Ho, Wo) == tuple(ref64.shape[2:])
    arena = E.Arena("h16")
    out = E.Act(torch.full((B, Ho, Wo, 64 + 8), 7.0, device="cuda"), 4, 64)
    for _ in range(2):                      # second call reuses the zero-bordered row planes
        layer(x.cuda(), out, arena, "t")
    err = float((out.to_nchw().cpu().double() - ref64).abs().max())
    print(shape, win, "stem max|err| vs fp64", err)
    assert err < 2e-5, err
    assert float(out.t[..., :4].min()) == 7.0 and float(out.t[..., 68:].min()) == 7.0


@pytest.mark.parametrize("shape", [(2, 3, 64, 96), (3, 3, 70, 154), (1, 3, 34, 30), (2, 3, 96, 320), (16, 3, 96, 160)])
def test_stem_with_fused_maxpool_is_bit_identical(shape):
    """conv1 + BN + ReLU + MaxPool2d(3, 2, 1) (R/backbones/resnet.py:186-189) in one kernel -- every 8 x 16 conv tile pooled in shared memory by the
    epilogue, windows that straddle tiles combined with atomicMax on the (non-negative) bit pattern -- against the stem kernel followed by the
    max-pool kernel: bit for bit (max is exact), including odd conv output sizes, partial tiles and more tiles than SMs; repeated calls agree
    (the border positions are re-zeroed by every launch); the pooled tensor respects its channel slice."""
    E = _E()
    B, C, H, W = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = (torch.randn(B, C, H, W, generator=g) * 2.0).cuda()
    w = torch.randn(64, C, 7, 7, generator=g) / np.sqrt(C * 49)
    bn = dict(weight=torch.rand(64, generator=g) + 0.5, bias=torch.randn(64, generator=g) * 0.3,
              running_mean=torch.randn(64, generator=g) * 0.1, running_var=torch.rand(64, generator=g) + 0.5)
    layer = E.StemLayer(w, bn, stride=2, pad=3, relu=True, device="cuda")
    Hs, Ws = layer.out_hw(H, W)
    Hp, Wp = (Hs - 1) // 2 + 1, (Ws - 1) // 2 + 1
    arena = E.Arena("h16")
    full = layer(x, E.Act(torch.empty(B, Hs, Ws, 64, device="cuda")), arena, "a")
    want = E.maxpool3x3s2(full, E.Act(torch.empty(B, Hp, Wp, 64, device="cuda")))
    assert torch.equal(want.to_nchw(), F.max_pool2d(full.to_nchw(), 3, 2, 1))
    got = E.Act(torch.full((B, Hp, Wp, 64 + 8), 7.0, device="cuda"), 4, 64)
    for _ in range(2):
        layer(x, got, arena, "b", pool=True)
        torch.cuda.synchronize()
        assert torch.equal(got.t[..., 4:68], want.t), float((got.t[..., 4:68] - want.t).abs().max())
    assert float(got.t[..., :4].min()) == 7.0 and float(got.t[..., 68:].min()) == 7.0
    assert float(want.t.min()) >= 0.0 and float((want.t == 0).float().mean()) < 0.9


@pytest.mark.parametrize("shape", [(2, 3, 64, 96), (3, 3, 70, 154), (1, 3, 34, 30), (2, 3, 96, 320), (16, 3, 96, 160), (2, 3, 384, 1280), (1, 3, 75, 515), (5, 3, 21, 1010)])
@pytest.mark.parametrize("f32_out", [True, False])
def test_stem_row_strip_kernel_is_bit_identical(shape, f32_out):
    """stem_pool_kernel in csrc/row_conv.cu (conv1 + BN + ReLU + MaxPool2d(3, 2, 1) as one row-strip kernel: overlapping windows through a no-swizzle wgmma
    descriptor, max-pool in registers, pooled tensor as fp16 planes [+ fp32]) against the stem kernel followed by the max-pool kernel: bit for
    bit, for one and several strips / row segments, odd conv and pooled sizes, image rows above / below the image, a channel slice, repeated calls."""
    E = _E()
    B, C, H, W = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = (torch.randn(B, C, H, W, generator=g) * 2.0).cuda()
    w = torch.randn(64, C, 7, 7, generator=g) / np.sqrt(C * 49)
    bn = dict(weight=torch.rand(64, generator=g) + 0.5, bias=torch.randn(64, generator=g) * 0.3,
              running_mean=torch.randn(64, generator=g) * 0.1, running_var=torch.rand(64, generator=g) + 0.5)
    layer = E.StemLayer(w, bn, stride=2, pad=3, relu=True, device="cuda")
    assert layer.row_kernel_ok()
    Hs, Ws = layer.out_hw(H, W)
    Hp, Wp = (Hs - 1) // 2 + 1, (Ws - 1) // 2 + 1
    arena = E.Arena("h16")
    full = layer(x, E.Act(torch.empty(B, Hs, Ws, 64, device="cuda")), arena, "a")
    want = E.maxpool3x3s2(full, E.Act(torch.empty(B, Hp, Wp, 64, device="cuda")))
    wh = want.t.half()
    wl = (want.t - wh.float()).half()
    got = E.Act(torch.full((B, Hp, Wp, 64 + 16), 7.0, device="cuda"), 8, 64, torch.full((2, B, Hp, Wp, 64 + 16), 3.0, device="cuda", dtype=torch.float16))
    for _ in range(2):
        r = layer(x, got, arena, "b", pool=True, f32_out=f32_out)
        torch.cuda.synchronize()
        assert layer.wrote_planes and r.f32 == f32_out
        assert torch.equal(got.lo[0][..., 8:72], wh) and torch.equal(got.lo[1][..., 8:72], wl), float((got.lo[0][..., 8:72].float() - wh.float()).abs().max())
        if f32_out:
            assert torch.equal(got.t[..., 8:72], want.t), float((got.t[..., 8:72] - want.t).abs().max())
        else:
            assert float(got.t.min()) == 7.0 and float(got.t.max()) == 7.0
    assert float(got.t[..., :8].min()) == 7.0 and float(got.t[..., 72:].min()) == 7.0
    assert float(got.lo[..., :8].float().min()) == 3.0 and float(got.lo[..., 72:].float().max()) == 3.0


ROW_CONV_CASES = [
    # B, Cin, pc, H, W, Cout, k, stride, pad
    (2, 3, 8, 40, 150, 16, 7, 1, 3),        # DLA base_layer: 7x7, image as 8-channel planes
    (1, 3, 8, 96, 320, 16, 7, 1, 3),
    (2, 16, 16, 33, 141, 16, 3, 1, 1),      # level0: 16-channel planes, every second operand row is an output column
    (1, 16, 16, 64, 640, 16, 3, 1, 1),
    (2, 16, 16, 33, 141, 32, 3, 2, 1),      # level1: stride 2, every fourth operand row
    (3, 16, 16, 96, 320, 32, 3, 2, 1),
    (1, 3, 8, 384, 1280, 16, 7, 1, 3),      # full size: 10 strips, several row segments
    (2, 3, 4, 40, 150, 16, 7, 2, 3),        # the ResNet stem's conv geometry: 4-channel planes, 7x7 / 2, two K steps per filter row
    (2, 3, 4, 40, 150, 32, 7, 2, 3),
]


@pytest.mark.parametrize("case", ROW_CONV_CASES)
def test_row_conv_vs_fp64(case):
    """csrc/row_conv.cu (few-channel convs as row-strip wgmma kernels: overlapping windows through a no-swizzle wgmma descriptor on fp16 (hi, lo)
    row planes) against an fp64 convolution of the same fp32 inputs: < 2e-5 (the bound of the fp16-split engine), fp32 output and planes, output
    written at a column offset of a wider, zero-bordered buffer (the next row conv's input form), neighbouring channels untouched."""
    E = _E()
    B, Cin, pc, H, W, Cout, k, s, p = case
    g = torch.Generator().manual_seed(sum(case))
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / np.sqrt(Cin * k * k)
    bn = dict(weight=torch.rand(Cout, generator=g) + 0.5, bias=torch.randn(Cout, generator=g) * 0.3,
              running_mean=torch.randn(Cout, generator=g) * 0.1, running_var=torch.rand(Cout, generator=g) + 0.5)
    layer = E.RowConvLayer(w, bn, stride=s, pad=p, relu=True, pc_in=pc, device="cuda")
    xoff = p + (2 if pc == 4 else 1)
    Wp = layer.in_pitch(W, xoff)
    planes = torch.zeros(2, B, H, Wp, pc, dtype=torch.float16, device="cuda")
    if Cin <= 4 and pc in (4, 8):
        xin = E.image_to_row_planes(x.cuda(), planes, xoff)
    else:
        xh = x.half()
        xl = (x - xh.float()).half()
        planes[0, :, :, xoff:xoff + W, :Cin] = xh.permute(0, 2, 3, 1).cuda()
        planes[1, :, :, xoff:xoff + W, :Cin] = xl.permute(0, 2, 3, 1).cuda()
        xin = E.RowPlanes(planes, W, xoff)
    xq = (planes[0].float() + planes[1].float())[:, :, xoff:xoff + W, :Cin].permute(0, 3, 1, 2).double().cpu()      # what the kernel sees (22 significant bits)
    assert float((xq - x.double()).abs().max()) < 1e-6
    wf, bf = E.fold_bn(w, None, bn)
    ref = F.relu(F.conv2d(xq, wf.double(), bf.double(), stride=s, padding=p)).float()
    Ho, Wo = layer.out_hw(H, W)
    oW, oxo, cs, co = Wo + 5, 2, Cout + 16, 8
    of = torch.full((B, Ho, oW, cs), 7.0, device="cuda")
    op = torch.full((2, B, Ho, oW, cs), 3.0, device="cuda", dtype=torch.float16)
    for _ in range(2):
        layer(xin, op, of, out_xoff=oxo, out_co=co)
    torch.cuda.synchronize()
    got = of[:, :, oxo:oxo + Wo, co:co + Cout].permute(0, 3, 1, 2).cpu()
    err = float((got - ref).abs().max())
    print(case, "max|err|", err)
    assert err < 2e-5, err
    gp = (op[0].float() + op[1].float())[:, :, oxo:oxo + Wo, co:co + Cout].permute(0, 3, 1, 2).cpu()
    assert float((gp - got).abs().max()) < 2e-6 and torch.equal(op[0][:, :, oxo:oxo + Wo, co:co + Cout], of[:, :, oxo:oxo + Wo, co:co + Cout].half())
    assert float(of[..., :co].min()) == 7.0 and float(of[..., co + Cout:].min()) == 7.0 and float(of[:, :, :oxo].min()) == 7.0 and float(of[:, :, oxo + Wo:].min()) == 7.0
    assert float(op[..., :co].float().min()) == 3.0 and float(op[:, :, :, :oxo].float().max()) == 3.0 and float(op[:, :, :, oxo + Wo:].float().min()) == 3.0
    # planes-only output gives the same planes
    op2 = torch.full_like(op, 3.0)
    layer(xin, op2, None, out_xoff=oxo, out_co=co)
    torch.cuda.synchronize()
    assert torch.equal(op2, op)


@pytest.mark.parametrize("shape", [(2, 64, 6, 80, 24), (1, 128, 5, 37, 12), (3, 64, 3, 50, 32), (1, 64, 2, 20, 4), (2, 192, 4, 64, 8)])
def test_psm_cosine_tensor_core_vs_oracle(shape):
    """tensor-core PSMCosine (flat 128-pixel tiles x 160-pixel window, band extracted in the epilogue) against the oracle;
    shapes with npix not a multiple of 128, W < D + 32, two and three 64-channel k-blocks."""
    E = _E()
    B, C, H, W, D = shape
    g = torch.Generator().manual_seed(sum(shape))
    left, right = torch.randn(B, C, H, W, generator=g), torch.randn(B, C, H, W, generator=g)
    ref = tp.psm_cosine(left, right, D * 4, 4)
    f = E.Act(nhwc(torch.cat([left, right])).cuda(), 0, None, torch.zeros(2, 2 * B, H, W, C, device="cuda", dtype=torch.float16))
    out = E.Act(torch.full((B, H, W, D + 8), 7.0, device="cuda"), 4, D)
    E.psm_cosine_stereo(f, B, D, out, planes_fresh=False)
    got = out.to_nchw().cpu()
    err = float((got - ref).abs().max())
    print(shape, "max|err|", err)
    assert err < 5e-6, err
    assert torch.equal(got == 0, ref == 0) or float((got - ref).abs().max()) < 5e-6
    assert float(out.t[..., :4].min()) == 7.0 and float(out.t[..., 4 + D:].min()) == 7.0
    # the masked triangle (w < d) is exactly zero
    for d in range(1, D):
        assert float(got[:, d, :, :min(d, W)].abs().max()) == 0.0
