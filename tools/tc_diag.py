"""Diagnostics of the wgmma gather-GEMM (csrc/sparse_conv.cu: k_gather_gemm_tc) on structured inputs: which operand
layout is wrong shows in WHERE the output differs, not only that it does.  Needs a GPU; prints one JSON line per
case and writes tc_diag_out/<tag>_tc_diag.json.   usage: python tools/tc_diag.py [tag]"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nksr_b200.unet import gather_gemm, round_tf32  # noqa: E402


def tc(x, idx, w, bias=None, res=None, relu=False):
    return gather_gemm(x, idx, round_tf32(w).transpose(1, 2).contiguous(), bias, res, relu, tf32=3)


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else "dev"
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    out = []

    def record(name, got, ref, extra=None):
        err = float((got - ref).abs().max())
        scale = float(ref.abs().max()) + 1e-30
        bad = (got - ref).abs() > 4e-3 * scale
        rec = dict(case=name, max_err=err, scale=scale, rel=err / scale, bad_frac=float(bad.float().mean()),
                   finite=bool(torch.isfinite(got).all()))
        if bad.any():
            rows = torch.nonzero(bad.any(dim=1)).squeeze(1)
            cols = torch.nonzero(bad.any(dim=0)).squeeze(1)
            rec.update(bad_rows=rows[:16].tolist(), n_bad_rows=int(rows.numel()), bad_cols=cols[:64].tolist())
        if extra:
            rec.update(extra)
        out.append(rec)
        print(json.dumps(rec), flush=True)

    quick = os.environ.get("NKSR_TC_QUICK") == "1"          # only the wide-layer timing (+ the U-Net breakdown)
    for c_in, c_out in ([] if quick else [(32, 32), (32, 64), (64, 64), (128, 64), (32, 96)]):
        n = 300
        x = torch.randn((n, c_in), generator=g).to(dev)
        ident = torch.arange(n, dtype=torch.int32, device=dev)[:, None].contiguous()
        # 1. one tap, identity gather, W = [I | 0] or stacked identities: y[:, j] = x[:, j % c_in] -- A, D layouts
        w = torch.zeros((1, c_in, c_out))
        for j in range(c_out):
            w[0, j % c_in, j] = 1.0
        w = w.to(dev)
        ref = round_tf32(x)[:, [j % c_in for j in range(c_out)]]
        got = tc(x, ident, w)
        extra = None
        if c_in == c_out == 32 and not torch.allclose(got, ref, atol=2e-3):
            # where did column j of x go?  (row 5, a generic row)
            m = (got[5][None, :] - x[5][:, None]).abs() < 2e-3
            extra = dict(col_map_row5=[torch.nonzero(m[j]).squeeze(1).tolist() for j in range(32)])
        record(f"identity_{c_in}x{c_out}", got, ref, extra)
        # 2. one-hot rows: y[i] = W[0][i % c_in, :] -- B layout
        x1 = torch.zeros((n, c_in))
        x1[torch.arange(n), torch.arange(n) % c_in] = 1.0
        w2 = (torch.randn((1, c_in, c_out), generator=g)).to(dev)
        got = tc(x1.to(dev), ident, w2)
        record(f"onehot_{c_in}x{c_out}", got, round_tf32(w2)[0][torch.arange(n) % c_in])
        # 3. random, 27 taps with holes
        idx = torch.randint(-1, n, (1000, 27), generator=g).to(torch.int32).to(dev)
        w3 = (torch.randn((27, c_in, c_out), generator=g) / (27 * c_in) ** 0.5).to(dev)
        b = torch.randn(c_out, generator=g).to(dev)
        res = torch.randn((1000, c_out), generator=g).to(dev)
        ref = gather_gemm(x, idx, w3, b, res, True, impl="torch")
        record(f"random27_{c_in}x{c_out}", tc(x, idx, w3, b, res, True), ref)
    # timing at the U-Net's layer shapes (rows scaled to the cfg4 hierarchy's level sizes / 8) against the mma.sync kernel
    def ms_of(fn, reps=5):
        for _ in range(2):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    for n, c_in, c_out in [(100_000, 128, 128)] if quick else [(2_000_000, 32, 32), (2_000_000, 64, 32), (425_000, 64, 64), (425_000, 128, 64),
                           (100_000, 128, 128), (100_000, 256, 128), (25_000, 256, 256)]:
        x = torch.randn((n, c_in), device=dev)
        nb = (torch.arange(n, device=dev)[:, None] + torch.arange(-13, 14, device=dev)[None, :] * 37)
        idx = torch.where((nb >= 0) & (nb < n), nb, torch.full_like(nb, -1)).to(torch.int32).contiguous()
        w = torch.randn((27, c_in, c_out), device=dev) / (27 * c_in) ** 0.5
        wt, wr = round_tf32(w).transpose(1, 2).contiguous(), round_tf32(w)
        t_mma = ms_of(lambda: gather_gemm(x, idx, wr, None, None, True, tf32=2))
        t_tc = ms_of(lambda: gather_gemm(x, idx, wt, None, None, True, tf32=3))
        fl = 2 * n * 27 * c_in * c_out / 1e9
        a, b_ = gather_gemm(x, idx, wr, None, None, True, tf32=2), gather_gemm(x, idx, wt, None, None, True, tf32=3)
        rec = dict(case=f"time_{n}_{c_in}x{c_out}", ms_mma_sync=t_mma,
                   ms_wgmma=t_tc, tflops_mma_sync=fl / t_mma, tflops_wgmma=fl / t_tc,
                   gather_tb_s_wgmma=n * 27 * c_in * 4 * max(1, c_out // (128 if c_out % 128 == 0 else 64)) / t_tc / 1e9,
                   rel_diff=float((a - b_).abs().max() / a.abs().max()))
        out.append(rec)
        print(json.dumps(rec), flush=True)
        del x, nb, idx, a, b_
    # where the U-Net backbone's time goes: the convolutions (our kernel) against the torch glue around them
    if os.environ.get("NKSR_TC_UNET", "1") == "1":
        import numpy as np
        import nksr_b200.unet as U
        from nksr_b200.network import NKSRNetwork
        from nksr_b200.svh import SparseFeatureHierarchy
        from tests import scenes
        xyz, _, _ = scenes.crop("cfg4_outdoor", 1_000_000, with_sensor=True)
        pts = torch.from_numpy(np.ascontiguousarray(xyz)).to(dev)
        svh = SparseFeatureHierarchy(0.1, 4, dev).build_point_splatting(pts)
        net = NKSRNetwork(dict(backbone="unet", tree_depth=4, kernel_dim=4, precision="tc")).to(dev)
        feat = torch.nn.functional.normalize(torch.randn((pts.shape[0], 3), device=dev), dim=1)
        acc = {"ms": 0.0, "calls": 0, "ev": []}
        orig = U.gather_gemm

        def timed(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = orig(*a, **k)
            e1.record()
            acc["ev"].append((e0, e1))
            return r
        with torch.no_grad():
            enc = net.encoder(pts, feat, svh, 0)
            for mode in (3, True):
                net.backbone_net(enc.x0, svh, tf32=mode)
                total = ms_of(lambda: net.backbone_net(enc.x0, svh, tf32=mode), reps=3)
                U.gather_gemm = timed
                acc["ev"].clear()
                net.backbone_net(enc.x0, svh, tf32=mode)
                torch.cuda.synchronize()
                U.gather_gemm = orig
                conv = sum(a.elapsed_time(b) for a, b in acc["ev"])
                t_enc = ms_of(lambda: net.encoder(pts, feat, svh, 0), reps=3)
                rec = dict(case="unet_breakdown", mode="wgmma" if mode == 3 else "mma_sync",
                           voxels=[svh.num_voxels(l) for l in range(4)],
                           backbone_ms=total, conv_ms=conv, conv_calls=len(acc["ev"]), glue_ms=total - conv,
                           point_encoder_ms=t_enc)
                out.append(rec)
                print(json.dumps(rec), flush=True)
    os.makedirs("tc_diag_out", exist_ok=True)
    with open(f"tc_diag_out/{tag}_tc_diag.json", "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
