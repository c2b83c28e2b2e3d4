"""Pipeline timeline of the persistent tensor-core conv (CTA 0): per k-block clock64 stamps -> load latency, MMA-thread wait time, period.
usage: python tools/trace_conv.py [shape-index ...]   (shapes of tools/prof_conv.py)"""
import os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualdet3d_b200 import engine as E, _lib

SHAPES = [("head 1408->1408 @24x80 B8", 8, 24, 80, 1408, 1408), ("layer1 64->64 @96x320 B16", 16, 96, 320, 64, 64),
          ("layer2 128->128 @48x160 B16", 16, 48, 160, 128, 128), ("layer3 256->256 @24x80 B16", 16, 24, 80, 256, 256)]
sel = [int(a) for a in sys.argv[1:]] or [0, 1, 2, 3]
N = 600
g = torch.Generator().manual_seed(0)
lib = _lib.load()
for si in sel:
    name, B, H, W, Cin, Cout = SHAPES[si]
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / np.sqrt(Cin * 9)
    layer = E.ConvLayer(w, None, None, pad=1, relu=True, device="cuda", engine="tc16")
    x = E.Act(torch.randn(B, H, W, Cin, generator=g).cuda(), 0, None, torch.zeros(2, B, H, W, Cin, device="cuda", dtype=torch.float16))
    E.split_lo(x)
    out = E.Act(torch.zeros(B, H, W, Cout, device="cuda"), 0, None, torch.zeros(2, B, H, W, Cout, device="cuda", dtype=torch.float16))
    for bn in (int(v) for v in os.environ.get("TRACE_BNS", "0,128").split(",")):
        layer.bn_tile = bn
        layer(x, out); torch.cuda.synchronize()
        tr = torch.zeros(12, N, dtype=torch.int64, device="cuda")
        lib.vd3d_tc_set_trace(tr.data_ptr(), N)
        layer(x, out); torch.cuda.synchronize()
        lib.vd3d_tc_set_trace(None, 0)
        t = tr.cpu().numpy().astype(np.float64)
        # per tile (rows 5..8, 11): last MMAs done, staged and handed over, epilogue start, stage released, epilogue done; the next tile's
        # first MMAs start at k-block (i + 1) * KB of row 3
        KB = 9 * ((Cin + 63) // 64)
        nkb = int((t[3] > 0).sum())
        first = t[3, :nkb:KB]                                        # first MMAs of each tile
        if len(first) > 2:
            print(f"{name:30s} bn={bn:3d} tile period (first MMA to first MMA) {np.median(np.diff(first)):7.0f} clk", flush=True)
        nt = int((t[5] > 0).sum())
        if nt > 2 and (t[7, :nt] > 0).all():                        # (tiles of <= 64 columns run the epilogue on the consumers: no hand-off)
            ti = np.arange(nt - 1)
            last, staged, estart, erel, edone = t[5, ti], t[6, ti], t[7, ti], t[8, ti], t[11, ti]
            nxt = t[3, np.minimum((ti + 1) * KB, N - 1)]
            ok = (ti + 1) * KB < nkb
            med = lambda v: np.median(v[ok]) if ok.any() else float("nan")
            print(f"{name:30s} bn={bn:3d} tiles={nt} k-blocks/tile={KB}  tile period {np.median(np.diff(t[5, :nt])):7.0f}  "
                  f"last MMA -> staged {med(staged - last):6.0f}  staged -> epilogue start {med(estart - staged):6.0f}  "
                  f"stage held {med(erel - estart):6.0f}  epilogue {med(edone - estart):6.0f}  "
                  f"last MMA -> next tile's first MMA {med(nxt - last):6.0f} clk", flush=True)
        # per tile: ring slot of every k-block (row 9), the longest wait for a stage ([3] - [2]) and where it fell, how often the producer
        # passed over the held slot (row 10).  With the held slot passed over, no k-block after a tile's second should wait about as long
        # as the epilogue holds its stage.
        wait_kb = t[3, :nkb] - t[2, :nkb]
        late = []
        for i in range(min(nt, nkb // KB)):
            w = wait_kb[i * KB:(i + 1) * KB]
            if KB > 2:
                late.append(w[2:].max())
            if i < 6:
                sl = "".join(str(int(v)) for v in t[9, i * KB:(i + 1) * KB][:48]) + ("..." if KB > 48 else "")
                print(f"   tile {i:3d}: slots {sl}  longest stage wait {w.max():7.0f} clk at k-block {int(w.argmax()):3d}  "
                      f"held slot passed over {int(t[10, i])}x", flush=True)
        if late:
            print(f"{name:30s} bn={bn:3d} longest stage wait after a tile's second k-block: median over tiles {np.median(late):7.0f}, "
                  f"max {np.max(late):7.0f} clk; held slot passed over {int(t[10, :nt].sum())}x in {nt} tiles", flush=True)
        n = int((t[0] > 0).sum())
        t = t[:, :n]
        t0 = t[0, 0]
        lat = t[3] - t[0]                  # stage free -> its MMAs start
        wait = t[2] - t[3]                 # issue start -> look-ahead wait for the next stage starts (= first half of the MMAs issued)
        issue = t[4] - t[3]                # 12 MMAs + look-ahead (wait, fence, descriptors) + commit
        per = np.diff(t[4])
        sl = slice(20, min(n, 400))
        print(f"{name:30s} bn={bn:3d} n={n}  period {np.median(per[sl]):7.0f}  free->mma-start {np.median(lat[sl]):7.0f}  "
              f"issue-loads {np.median((t[1]-t[0])[sl]):5.0f}  half-issue {np.median(wait[sl]):7.0f}  mma-issue {np.median(issue[sl]):6.0f} clk", flush=True)
        k = 40
        print("   k-block:", " ".join(f"{int(v):6d}" for v in range(k, k + 8)))
        for r, lab in enumerate(["free", "issued", "lookahd", "mmastart", "mmadone"]):
            print(f"   {lab:8s}", " ".join(f"{int(v - t0):6d}" for v in t[r, k:k + 8]))
