"""-m gpu: the two op families the reference builds under make.sh (DCN v1/v2, iou3d) against (a) what the reference's OWN compiled
extensions (oracle/_ref, built by oracle/build_ref.py from the reference sources) return for the same seeded inputs, stored in
tests/golden/ref_ops.npz by tests/golden/make_golden_ref_ops.py, and (b) CPU restatements."""
import os

import numpy as np
import pytest
import torch

import torch_port as tp
from conftest import GOLDEN

pytestmark = pytest.mark.gpu
N_SAMPLE = 2048                  # stored values per large reference tensor (a fixed seeded sample of positions)
RECORD = {} if os.environ.get("VD3D_RECORD_REF") else None      # make_golden_ref_ops.py: run the real extensions and record
_STORED = {}


def sample(t):
    a = t.detach().reshape(-1).cpu().numpy()
    if a.size <= N_SAMPLE:
        return a
    return a[np.sort(np.random.default_rng(a.size).choice(a.size, N_SAMPLE, replace=False))]


def ref_out(key, run, full=False):
    """The reference extension's output `key` (flattened; sampled unless `full`; `key + "_absmax"` = max |.| of the whole tensor): from
    tests/golden/ref_ops.npz, or, while that file is being written, run(ext) on the real extension (ext(name) loads one)."""
    if RECORD is None:
        if not _STORED:
            _STORED.update(np.load(os.path.join(GOLDEN, "ref_ops.npz")))
        return _STORED[key]
    if run is not None:
        import build_ref
        t = run(build_ref.load)
        RECORD[key] = t.detach().reshape(-1).cpu().numpy() if full else sample(t)
        RECORD[key + "_absmax"] = np.float64(float(t.abs().max()))
    return RECORD[key]


def rand_boxes(n, g, spread=10.0):
    c = torch.rand(n, 2, generator=g) * spread
    wh = torch.rand(n, 2, generator=g) * 4 + 0.5
    ry = (torch.rand(n, generator=g) - 0.5) * 2 * np.pi
    return torch.cat([c - wh / 2, c + wh / 2, ry[:, None]], dim=1).contiguous()


def test_iou3d_pairwise_vs_reference_extension_and_clipping():
    from visualdet3d_b200.ops import iou3d
    g = torch.Generator().manual_seed(0)
    a, b = rand_boxes(70, g).cuda(), rand_boxes(45, g).cuda()

    def theirs(name):
        o2 = torch.zeros(70, 45, device="cuda")
        return lambda ext: (getattr(ext("ref_iou3d_cuda"), name)(a, b, o2), o2)[1]
    for mine, name in ((iou3d.boxes_overlap_bev_gpu, "boxes_overlap_bev_gpu"), (iou3d.boxes_iou_bev_gpu, "boxes_iou_bev_gpu")):
        o1 = torch.zeros(70, 45, device="cuda")
        assert mine(a, b, o1) == 1
        o2 = ref_out(name, theirs(name), full=True)
        torch.cuda.synchronize()
        np.testing.assert_allclose(o1.cpu().numpy().reshape(-1), o2, rtol=1e-4, atol=1e-5)
    ov = torch.zeros(70, 45, device="cuda")
    iou3d.boxes_overlap_bev_gpu(a, b, ov)
    ac, bc, ovc = a.cpu().numpy(), b.cpu().numpy(), ov.cpu().numpy()
    for i in range(0, 70, 7):
        for j in range(0, 45, 5):
            assert abs(ovc[i, j] - tp.rotated_overlap_bev(ac[i], bc[j])) < 2e-3, (i, j)
    # identical boxes: overlap == area, IoU == 1
    io = torch.zeros(70, 70, device="cuda")
    iou3d.boxes_iou_bev_gpu(a, a, io)
    np.testing.assert_allclose(torch.diagonal(io).cpu().numpy(), 1.0, atol=1e-3)


@pytest.mark.parametrize("n", [1, 63, 64, 65, 300])
def test_iou3d_nms_vs_reference_extension(n):
    from visualdet3d_b200.ops import iou3d
    g = torch.Generator().manual_seed(n)
    boxes = rand_boxes(n, g, spread=8.0).cuda()

    def theirs(name):
        k2 = torch.zeros(n, dtype=torch.int64)
        return lambda ext: k2[:getattr(ext("ref_iou3d_cuda"), name)(boxes, k2, 0.3)]
    for mine, name in ((iou3d.nms_gpu, "nms_gpu"), (iou3d.nms_normal_gpu, "nms_normal_gpu")):
        k1 = torch.zeros(n, dtype=torch.int64)
        n1, k2 = mine(boxes, k1, 0.3), ref_out(f"{name}_{n}", theirs(name), full=True)
        assert n1 == len(k2) and np.array_equal(k1[:n1].numpy(), k2)            # bit-exact keep indices
    assert iou3d.nms_gpu(boxes[:0], torch.zeros(0, dtype=torch.int64), 0.3) == 0
    with pytest.raises(RuntimeError):
        iou3d.nms_gpu(boxes.cpu(), torch.zeros(n, dtype=torch.int64), 0.3)


def test_boxes_iou3d_wrapper():
    from visualdet3d_b200.ops import iou3d
    g = torch.Generator().manual_seed(2)
    b = torch.rand(9, 7, generator=g) * 3 + 1
    b[:, 6] = (torch.rand(9, generator=g) - 0.5) * 3
    b = b.cuda()
    iou = iou3d.boxes_iou3d_gpu(b, b)
    np.testing.assert_allclose(torch.diagonal(iou).cpu().numpy(), 1.0, atol=1e-3)
    assert float(iou.max()) <= 1.0 + 1e-3 and float(iou.min()) >= 0.0


DCN_CASES = [  # B, C, H, W, Cout, k, stride, pad, dil, dg
    (2, 64, 20, 30, 64, 3, 1, 1, 1, 1),
    (1, 32, 17, 23, 48, 3, 1, 1, 1, 1),
    (2, 64, 12, 16, 32, 3, 2, 1, 1, 1),
    (1, 64, 10, 14, 64, 3, 1, 2, 2, 2),
    (1, 16, 9, 11, 24, 1, 1, 0, 1, 1),
]


@pytest.mark.parametrize("case", DCN_CASES)
def test_modulated_deform_conv_vs_reference_extension(case):
    from visualdet3d_b200.ops import dcn
    B, C, H, W, Co, k, s, p, d, dg = case
    g = torch.Generator().manual_seed(sum(case))
    x = torch.randn(B, C, H, W, generator=g)
    w = torch.randn(Co, C, k, k, generator=g) / np.sqrt(C * k * k)
    bias = torch.randn(Co, generator=g)
    Ho, Wo = (H + 2 * p - (d * (k - 1) + 1)) // s + 1, (W + 2 * p - (d * (k - 1) + 1)) // s + 1
    off = torch.randn(B, 2 * k * k * dg, Ho, Wo, generator=g) * 2.0
    off[0, :, 0, 0] = 50.0                 # far outside -> contributes zero
    off[0, :, 1, 1] = -0.999               # the `> -1` knife edge
    mask = torch.sigmoid(torch.randn(B, k * k * dg, Ho, Wo, generator=g))
    xc, wc, bc, oc, mc = x.cuda(), w.cuda(), bias.cuda(), off.cuda(), mask.cuda()
    out = torch.empty(B, Co, Ho, Wo, device="cuda")
    dcn.modulated_deform_conv_forward(xc, wc, bc, xc.new_empty(0), oc, mc, out, xc.new_empty(0), k, k, s, s, p, p, d, d, 1, dg, True)
    out_ref = torch.empty(B, Co, Ho, Wo, device="cuda")
    key = f"dcn_v2_{DCN_CASES.index(case)}"
    out_ref = ref_out(key, lambda ext: (ext("ref_deform_conv_ext").modulated_deform_conv_forward(
        xc, wc, bc, xc.new_empty(0), oc, mc, out_ref, xc.new_empty(0), k, k, s, s, p, p, d, d, 1, dg, True), out_ref)[1])
    torch.cuda.synchronize()
    np.testing.assert_allclose(sample(out), out_ref, rtol=1e-4, atol=2e-5)
    if dg == 1:
        cpu = tp.modulated_deform_conv(x, off, mask, w, bias, s, p, d)
        np.testing.assert_allclose(out.cpu().numpy(), cpu.numpy(), rtol=1e-4, atol=2e-5)
    # DCN v1 (no mask, no bias)
    o1 = torch.empty(B, Co, Ho, Wo, device="cuda"); o2 = torch.empty(B, Co, Ho, Wo, device="cuda")
    assert dcn.deform_conv_forward(xc, wc, oc, o1, xc.new_empty(0), xc.new_empty(0), k, k, s, s, p, p, d, d, 1, dg, B) == 1
    o2 = ref_out(key.replace("v2", "v1"), lambda ext: (ext("ref_deform_conv_ext").deform_conv_forward(
        xc, wc, oc, o2, xc.new_empty(0), xc.new_empty(0), k, k, s, s, p, p, d, d, 1, dg, B), o2)[1])
    torch.cuda.synchronize()
    np.testing.assert_allclose(sample(o1), o2, rtol=1e-4, atol=2e-5)


@pytest.mark.parametrize("case", DCN_CASES)
def test_deform_conv_backward_vs_reference_extension(case):
    """SURVEY.md 8(f) rank 4: the three backward entries of `deform_conv_ext` against the reference's own compiled kernels
    (modulated col2im / col2im_coord, deform_conv_cuda_kernel.cu:635-767; DCNv1 :279-436) on the same tensors: grad_input, grad_offset,
    grad_mask, grad_weight, grad_bias.  Sums run in a different order (one fused pass, fp32 atomics): rtol 1e-4 of the tensor's scale."""
    from visualdet3d_b200.ops import dcn
    B, C, H, W, Co, k, s, p, d, dg = case
    g = torch.Generator().manual_seed(1000 + sum(case))
    x = torch.randn(B, C, H, W, generator=g)
    w = torch.randn(Co, C, k, k, generator=g) / np.sqrt(C * k * k)
    bias = torch.randn(Co, generator=g)
    Ho, Wo = (H + 2 * p - (d * (k - 1) + 1)) // s + 1, (W + 2 * p - (d * (k - 1) + 1)) // s + 1
    off = torch.randn(B, 2 * k * k * dg, Ho, Wo, generator=g) * 2.0
    off[0, :, 0, 0] = 50.0
    mask = torch.sigmoid(torch.randn(B, k * k * dg, Ho, Wo, generator=g))
    gout = torch.randn(B, Co, Ho, Wo, generator=g)
    xc, wc, bc, oc, mc, gc = x.cuda(), w.cuda(), bias.cuda(), off.cuda(), mask.cuda(), gout.cuda()
    e = lambda: xc.new_empty(0)
    ci = DCN_CASES.index(case)

    def close(a, b, what, factor=1.0):           # b: the reference tensor's key; scale = max |.| of the whole reference tensor
        ref = ref_out(f"dcn_bwd_{ci}_{b[0]}", b[1]).astype(np.float64) * factor
        scale = float(ref_out(f"dcn_bwd_{ci}_{b[0]}_absmax", None)) * factor + 1e-12
        err = float(np.abs(sample(a).astype(np.float64) - ref).max()) / scale
        assert err < 1e-4, (what, err)
        return err

    def run_ref(v1):
        def run(ext):
            if "grads" not in memo:
                ref = ext("ref_deform_conv_ext")
                gi, gw, gb = torch.zeros_like(xc), torch.zeros_like(wc), torch.zeros_like(bc)
                go, gm = torch.zeros_like(oc), torch.zeros_like(mc)
                ref.modulated_deform_conv_backward(xc, wc, bc, e(), oc, mc, e(), gi, gw, gb, go, gm, gc, k, k, s, s, p, p, d, d, 1, dg, True)
                g1i, g1o, g1w = torch.zeros_like(xc), torch.zeros_like(oc), torch.zeros_like(wc)
                ref.deform_conv_backward_input(xc, oc, gc, g1i, g1o, wc, e(), k, k, s, s, p, p, d, d, 1, dg, B)
                ref.deform_conv_backward_parameters(xc, oc, gc, g1w, e(), e(), k, k, s, s, p, p, d, d, 1, dg, 0.5, B)
                torch.cuda.synchronize()
                memo["grads"] = (gi, gw, gb, go, gm, g1i, g1o, g1w)
            return memo["grads"][v1]
        return run
    memo = {}
    names = ("grad_input", "grad_weight", "grad_bias", "grad_offset", "grad_mask", "v1_grad_input", "v1_grad_offset", "v1_grad_weight")
    ref = {n: (n, run_ref(i)) for i, n in enumerate(names)}

    # ---- DCNv2 ----
    gi, gw, gb = torch.zeros_like(xc), torch.zeros_like(wc), torch.zeros_like(bc)
    go, gm = torch.zeros_like(oc), torch.zeros_like(mc)
    dcn.modulated_deform_conv_backward(xc, wc, bc, e(), oc, mc, e(), gi, gw, gb, go, gm, gc, k, k, s, s, p, p, d, d, 1, dg, True)
    torch.cuda.synchronize()
    res = (gi, gw, gb, go, gm)
    errs = [close(a, ref[n], n) for a, n in zip(res, names[:5])]
    # accumulate-into contracts: a second call doubles grad_input / grad_weight / grad_bias, re-assigns grad_offset / grad_mask
    gi, gw, gb, go, gm = [t.clone() for t in res]
    dcn.modulated_deform_conv_backward(xc, wc, bc, e(), oc, mc, e(), gi, gw, gb, go, gm, gc, k, k, s, s, p, p, d, d, 1, dg, True)
    close(gi, ref["grad_input"], "grad_input x2", 2.0), close(gw, ref["grad_weight"], "grad_weight x2", 2.0), close(go, ref["grad_offset"], "grad_offset again")
    # ---- DCNv1 ----
    gi, go, gw = torch.zeros_like(xc), torch.zeros_like(oc), torch.zeros_like(wc)
    assert dcn.deform_conv_backward_input(xc, oc, gc, gi, go, wc, e(), k, k, s, s, p, p, d, d, 1, dg, B) == 1
    assert dcn.deform_conv_backward_parameters(xc, oc, gc, gw, e(), e(), k, k, s, s, p, p, d, d, 1, dg, 0.5, B) == 1
    torch.cuda.synchronize()
    errs += [close(a, ref[n], n) for a, n in zip((gi, go, gw), names[5:])]
    print(case, "max relative errors", ["%.1e" % v for v in errs])


@pytest.mark.parametrize("case", [(2, 64, 24, 40, 64, 1, 1, 0.5), (1, 128, 20, 28, 64, 1, 1, 0.5), (2, 64, 17, 23, 256, 1, 1, 0.5), (1, 64, 21, 30, 128, 2, 1, 0.5),
                                  (1, 192, 9, 50, 96, 1, 2, 0.5), (2, 64, 33, 47, 64, 1, 1, 5.0), (1, 256, 13, 21, 128, 1, 1, 2.0)])
def test_fused_deform_conv_matches_unfused_and_reference(case, monkeypatch):
    """csrc/dcn_fused.cu (bilinear gather written straight into the swizzled shared-memory operand of the wgmma GEMM) against
    (a) the unfused path (fp16 column planes in HBM + 1x1 conv): bit-identical, same K order and gather arithmetic;
    (b) the reference's own compiled extension on the same tensors: rtol 1e-4."""
    from visualdet3d_b200 import engine as E
    B, C, H, W, Co, s, d, off_scale = case          # off_scale: spread of the offsets in pixels (5.0: most samples leave the staged halo -> global fallback)
    g = torch.Generator().manual_seed(int(sum(case)))
    x = torch.randn(B, C, H, W, generator=g)
    w = torch.randn(Co, C, 3, 3, generator=g) / np.sqrt(C * 9)
    bias = torch.randn(Co, generator=g)
    ow = torch.randn(27, C, 3, 3, generator=g) * 0.03
    ob = torch.randn(27, generator=g) * off_scale
    layer = E.DeformConvLayer(w, bias, ow, ob, None, stride=s, pad=d, dil=d, relu=True, device="cuda")
    assert layer.k_order == (1 if (s == 1 and d == 1) else 0)
    Ho, Wo = layer.out_hw(H, W)
    planes = lambda *sh: torch.zeros(2, *sh, device="cuda", dtype=torch.float16)
    xa = E.split_lo(E.Act(x.permute(0, 2, 3, 1).contiguous().cuda(), 0, None, planes(B, H, W, C)))
    res = E.Act(torch.randn(B, Ho, Wo, Co, generator=g).cuda())
    outs = []
    variants = [("1", "1"), ("0", "1")] + ([("1", "0")] if C == 64 else [])       # (fused, staged): staged fused / unfused / global-gather fused
    for fused, staged_env in variants:
        monkeypatch.setenv("VD3D_DCN_FUSED", fused)
        monkeypatch.setenv("VD3D_DCN_STAGED", staged_env)
        assert layer.fused_ok() == (fused == "1")
        ar = E.Arena()
        out = E.Act(torch.full((B, Ho, Wo, Co + 8), 7.0, device="cuda"), 4, Co, planes(B, Ho, Wo, Co + 8))
        layer(xa, out, ar, "t", res=res)
        torch.cuda.synchronize()
        outs.append((out.t.clone(), out.lo.clone(), ar))
    for o in outs[1:]:
        assert torch.equal(outs[0][0], o[0]) and torch.equal(outs[0][1], o[1])                    # fp32 output and its fp16 planes, bit for bit
    assert "dcn.cols" not in {k[0] for k in outs[0][2]._bufs} and "dcn.cols" in {k[0] for k in outs[1][2]._bufs}      # no column tensor in the fused path
    assert float(outs[0][0][..., :4].min()) == 7.0 and float(outs[0][0][..., 4 + Co:].min()) == 7.0   # channel slice respected
    # reference extension: offsets / mask from the same offset conv, computed by torch
    om = torch.nn.functional.conv2d(x, ow, ob, stride=s, padding=d, dilation=d)
    off, mask = om[:, :18].contiguous().cuda(), torch.sigmoid(om[:, 18:]).contiguous().cuda()
    xc = x.cuda()
    out_ref = torch.empty(B, Co, Ho, Wo, device="cuda")
    out_ref = ref_out(f"fused_{int(2 * sum(case))}", lambda ext: (ext("ref_deform_conv_ext").modulated_deform_conv_forward(
        xc, w.cuda(), bias.cuda(), xc.new_empty(0), off, mask, out_ref, xc.new_empty(0), 3, 3, s, s, d, d, d, d, 1, 1, True), out_ref)[1])
    want = np.maximum(out_ref + sample(res.t.permute(0, 3, 1, 2)), 0.0)
    got = outs[0][0][..., 4:4 + Co].permute(0, 3, 1, 2)
    np.testing.assert_allclose(sample(got), want, rtol=1e-4, atol=5e-5)


def test_dcn_error_behaviour_and_pack_module():
    from visualdet3d_b200.ops import dcn
    x = torch.randn(1, 32, 8, 8)
    w = torch.randn(16, 32, 3, 3)
    with pytest.raises(RuntimeError):
        dcn.modulated_deform_conv_forward(x, w, None, x, torch.zeros(1, 18, 8, 8), torch.ones(1, 9, 8, 8), torch.empty(1, 16, 8, 8), x,
                                          3, 3, 1, 1, 1, 1, 1, 1, 1, 1, False)
    with pytest.raises(RuntimeError):       # backward entries mirror the forward's checks (CPU tensors are refused, not computed on the host)
        dcn.modulated_deform_conv_backward(x, w, None, x, torch.zeros(1, 18, 8, 8), torch.ones(1, 9, 8, 8), x, torch.zeros_like(x), torch.zeros_like(w),
                                           None, torch.zeros(1, 18, 8, 8), torch.zeros(1, 9, 8, 8), torch.zeros(1, 16, 8, 8),
                                           3, 3, 1, 1, 1, 1, 1, 1, 1, 1, False)
    # module mirror vs the CPU restatement, conv_offset re-randomised (the reference zero-fills it)
    m = dcn.ModulatedDeformConvPack(64, 64, 3, padding=1)
    g = torch.Generator().manual_seed(0)
    m.conv_offset.weight.data = torch.randn(m.conv_offset.weight.shape, generator=g) * 0.05
    m.conv_offset.bias.data = torch.randn(27, generator=g) * 0.1
    sd = {"d." + k: v.detach().clone() for k, v in m.state_dict().items()}
    assert sorted(sd) == ["d.bias", "d.conv_offset.bias", "d.conv_offset.weight", "d.weight"]
    xin = torch.randn(2, 64, 14, 18, generator=g)
    ref = tp.modulated_deform_conv_pack(sd, "d", xin, 1, 1, 1)
    got = m.cuda()(xin.cuda()).cpu()
    np.testing.assert_allclose(got.numpy(), ref.numpy(), rtol=1e-4, atol=5e-5)
