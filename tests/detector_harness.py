"""Helpers shared by the detector GPU tests: a forward that captures every stage-hook tensor, and the two detection matchers (anchor
detectors against the oracle's anchor indices, CenterNet detectors against its peak indices)."""
import numpy as np
import torch


def run_with_stages(det, *inputs, flatten_heads=False):
    """`det.forward_batch(*inputs)` on the GPU with every stage-hook tensor captured (NCHW, on the host) -> (results, stages).
    flatten_heads: reshape the anchor heads' `cls_preds` / `reg_preds` to the reference's [B, N, C] / [B, N, 12]."""
    from visualdet3d_b200.engine import Act
    st = {}

    def hook(name, v):
        st[name] = v.to_nchw().cpu() if isinstance(v, Act) else v.detach().cpu().clone()
    det.stage_hook = hook
    try:
        with torch.no_grad():
            res = det.forward_batch(*[t.cuda() for t in inputs])
    finally:
        det.stage_hook = None
    if flatten_heads:
        B = inputs[0].shape[0]
        st["cls_preds"] = st["cls_preds"].permute(0, 2, 3, 1).reshape(B, -1, det.num_cls_output)
        st["reg_preds"] = st["reg_preds"].permute(0, 2, 3, 1).reshape(B, -1, 12)
    return res, st


def assert_dets_match(got, ref, got_anchor, atol=1e-3):
    """got = (scores, boxes, cls) from the CUDA path, ref = oracle (scores, boxes, cls, anchor_idx).  The kept ANCHOR SET must
    be identical; the row order must be identical except between rows whose scores are within 1e-5 of each other
    (a descending sort of scores that differ by an ulp between host and device libm); values within `atol`."""
    s, bx, ci = [t.cpu() for t in got]
    rs, rb, rc, ridx = ref
    ga = got_anchor.cpu().long()
    assert len(s) == len(rs), (len(s), len(rs))
    if len(s) == 0:
        return 0
    assert torch.equal(torch.sort(ga)[0], torch.sort(ridx)[0]), "kept anchor sets differ"
    swaps = 0
    if not torch.equal(ga, ridx):
        pos = {int(a): i for i, a in enumerate(ridx.tolist())}
        perm = torch.tensor([pos[int(a)] for a in ga.tolist()])
        moved = (perm != torch.arange(len(perm))).nonzero()[:, 0]
        swaps = len(moved)
        for i in moved.tolist():
            assert abs(float(rs[perm[i]]) - float(rs[i])) < 1e-5, "order differs between rows that are not score-tied"
        rs, rb, rc = rs[perm], rb[perm], rc[perm]
    assert torch.equal(ci, rc)
    assert float((s - rs).abs().max()) < atol, float((s - rs).abs().max())
    assert float((bx - rb).abs().max()) < atol, float((bx - rb).abs().max())
    return swaps


def match_dets(got, ref, got_index, atol=1e-3):
    """same peak set; same order except between score-tied rows; values within atol (boxes rtol 1e-5 on top)."""
    s, bx, ci = [t.cpu() for t in got]
    rs, rb, rc, rflat = ref
    assert len(s) == len(rs), (len(s), len(rs))
    if len(s) == 0:
        return
    gi = got_index.cpu().long()
    assert torch.equal(torch.sort(gi)[0], torch.sort(rflat)[0]), "kept peak sets differ"
    if not torch.equal(gi, rflat):
        pos = {int(a): i for i, a in enumerate(rflat.tolist())}
        perm = torch.tensor([pos[int(a)] for a in gi.tolist()])
        for i in (perm != torch.arange(len(perm))).nonzero()[:, 0].tolist():
            assert abs(float(rs[perm[i]]) - float(rs[i])) < 1e-5
        rs, rb, rc = rs[perm], rb[perm], rc[perm]
    assert ci.shape == rc.shape and torch.equal(ci, rc)
    assert float((s - rs).abs().max()) < atol
    np.testing.assert_allclose(bx.numpy(), rb.numpy(), atol=atol, rtol=1e-5)
