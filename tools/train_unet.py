"""Train the sparse-conv U-Net backbone (NKSRNetwork(backbone='unet', trainable=True)) on a seeded synthetic scene with
the structure and UDF losses (nksr_b200/training.py), Adam lr 1e-4, gradient norm clipped to 0.5 (train.yaml).

    python tools/train_unet.py --scene sphere --points 200000 --steps 30 --precision fp32 --out ckpt.pt
    python tools/train_unet.py --scene cfg4 --points 1000000 --depth 4 --precision tc --steps 10
    python tools/train_unet.py --scene cfg4 --points 1000000 --depth 4 --kernel-losses --steps 10
    python tools/train_unet.py --scene cfg4 --points 1000000 --depth 4 --structure predicted --steps 10
    python tools/train_unet.py --scene cfg4 --points 1000000 --depth 4 --udf --steps 10
    python tools/train_unet.py --scene sphere --points 200000 --depth 4 --geometry neural --steps 30
    python tools/train_unet.py --scene cfg4 --points 1000000 --depth 4 --kernel-losses --vol-sup --steps 10
    python tools/train_unet.py --scene cfg4 --points 1000000 --depth 4 --kernel-losses --operator matrix_free --steps 10
    python tools/train_unet.py --scene sphere --mesh-gt --mesh-scan --steps 10

Scenes: 'sphere' (tests/clouds.py, exact normals) or 'cfg4' (a crop of bench.py's outdoor scene at its own density,
normals from the kNN preprocess).  Every step prints one JSON line: the losses and the CUDA-event times of the forward,
the backward (with the sparse convolution's input-gradient and weight-gradient kernels separately) and the optimizer
step.  The last line is a summary over the steps after the first two: median times, the weight-gradient kernel's
achieved TFLOP/s (2 nnz_taps c_in c_out per call) and GB/s per (c_in, c_out) shape, and the GPU's name and power limit.
--kernel-losses adds the kernel-field losses (GT-surface value / normal, spatial TSDF), trained through the kernel solve,
and reports them per step with the CUDA-event times of the forward solve (assembly + PCG), the adjoint PCG and the VJP
kernels (with the field evaluations they need).  --operator matrix_free runs both PCGs on the matrix-free operator
(no Gram matrix); the solve time then sums the kernel rows, the operator setup and the PCG.
--structure predicted grows the decoder hierarchy from the structure head (teacher-forced from the ground truth, or
from the prediction with probability --pd-structure-prob); after training one more line reports, per level, the
structure accuracy and the sizes |E_l| (encoder), |T_l| (grown) and |dec_l| (kept), the CUDA-event time of every growth
step and the backbone's forward time on the encoder hierarchy against the grown one under teacher forcing.
--geometry neural builds the network with geometry='neural': the field losses (implied) are taken on the NeuralField
output field sdf_decoder(u(x)), whose normal loss trains through its position gradient (no solve).
--udf builds the network with udf.enabled: the UDF loss is the NeuralField's over every level of the decoder hierarchy,
through the interpolation kernels (csrc/neural_field.cu), instead of the finest level's alone.
--vol-sup (cfg4 only) trains with volume ground truth, the reference's default supervision: a PointTSDFVolume built from
the crop's sensor rays (csrc/tsdf_volume.cu, DESIGN.md SPEC S19) with node spacing h = W, truncation tau = 2 W and a
margin of one top-level voxel around the points -- our choices, the reference ships its volumes as data.  The setup
line reports the build time and the near / free / unknown fractions of the nodes; with --kernel-losses every step
reports the spatial loss's empty-space term (spatial_empty).
--mesh-gt (sphere only) trains against a mesh: MeshGroundTruth (DESIGN.md SPEC S21) of a level-6 icosphere (81,920
triangles) of the scene's radius 0.35, tau = 2 W, its SDF the exact distance to the triangles signed by ray parity.
--mesh-scan (with --mesh-gt) takes the input from a simulated LiDAR scan of that icosphere instead of the analytic
sphere: a ring of 8 sensors at radius 1 around it, alternately 0.3 above and below its equator, each casting
lidar_directions(128, n_azimuth, (-37, 37)) with n_azimuth chosen for about --points returns (gt_geometry.scan_mesh,
SPEC S22); the points then take the kNN normal preprocess with the sensor flip (64 neighbours, 85 degrees), as
examples/recons_waymo.py does.  The setup line reports the scan's rays, returns and time.
--out saves {'state_dict': ...}, which load_checkpoint_from_url(<path>) + load_state_dict take."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")


def cfg4_crop(n, device):
    """points, normals and sensor positions of an n-point cfg4 crop after get_estimate_normal_preprocess_fn(64, 85.0)
    (kNN normals, grazing-angle filter), and the voxel size"""
    import torch
    from nksr_b200 import _lib
    from nksr_b200.reconstructor import estimate_normals_knn
    from tests import scenes
    xyz, sensor, W = scenes.crop("cfg4_outdoor", n, with_sensor=True)
    r = estimate_normals_knn(torch.from_numpy(xyz).to(device), torch.from_numpy(sensor).to(device), 64, 85.0)
    scan = _lib.exclusive_scan32(r.keep)
    cnt = int(scan[-1].item())
    px, pn, ps = (_lib.compact_rows(a, r.keep, scan, cnt) for a in (r.xyz, r.normal, r.sensor))
    return px, pn, ps, W


def build_volume(px, pn, ps, W, depth):
    """the volume ground truth of --vol-sup: h = W, tau = 2 W, a margin of one top-level voxel"""
    from nksr_b200.gt_geometry import PointTSDFVolume
    return PointTSDFVolume.from_sensor_rays(px, pn, ps, h=W, tau=2.0 * W, margin=W * 2 ** (depth - 1))


MESH_GT_LEVEL = 6       # --mesh-gt: 81,920 triangles, the size of a ShapeNet model


def build_mesh_gt(W, device):
    """the mesh ground truth of --mesh-gt: an icosphere of radius 0.35 (tests.clouds.sphere's), tau = 2 W"""
    import torch
    from nksr_b200.gt_geometry import MeshGroundTruth
    from tests.test_cpu_occupancy import icosphere
    v, f = icosphere(MESH_GT_LEVEL, 0.35)
    return MeshGroundTruth(torch.from_numpy(v).to(device), torch.from_numpy(f).to(device), tau=2.0 * W)


SCAN_SENSORS, SCAN_BEAMS, SCAN_ELEVATION = 8, 128, (-37.0, 37.0)   # --mesh-scan: the sphere spans about +-20 degrees


def scan_input(gt, n, device):
    """the input of --mesh-scan: points of a simulated scan of gt's mesh after the kNN normal preprocess with the
    sensor flip, their normals, and the scan's statistics"""
    import math
    import torch
    from nksr_b200 import _lib
    from nksr_b200.gt_geometry import lidar_directions, scan_mesh
    from nksr_b200.reconstructor import estimate_normals_knn
    a = 2.0 * math.pi * torch.arange(SCAN_SENSORS, dtype=torch.float64) / SCAN_SENSORS
    z = 0.3 * (1.0 - 2.0 * (torch.arange(SCAN_SENSORS) % 2))
    sensors = torch.stack([torch.cos(a), torch.sin(a), z], dim=1).float()
    # about 4.5 % of the rays of each sensor meet the sphere
    n_azimuth = max(64, int(round(n / (0.045 * SCAN_SENSORS * SCAN_BEAMS))))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    scan = scan_mesh(gt.mesh, sensors, lidar_directions(SCAN_BEAMS, n_azimuth, SCAN_ELEVATION))
    e1.record()
    r = estimate_normals_knn(scan.xyz, scan.sensor, 64, 85.0)
    s = _lib.exclusive_scan32(r.keep)
    cnt = int(s[-1].item())
    px, pn = (_lib.compact_rows(x, r.keep, s, cnt) for x in (r.xyz, r.normal))
    torch.cuda.synchronize()
    return px, pn, dict(rays=SCAN_SENSORS * SCAN_BEAMS * n_azimuth, returns=int(scan.xyz.shape[0]), kept=cnt,
                        scan_ms=round(e0.elapsed_time(e1), 3))


def make_scene(kind, n, depth, device, vol_sup=False, mesh_gt=False, mesh_scan=False):
    """the TrainingScene, and with vol_sup the volume's grid, build time (ms) and class fractions; with mesh_gt the
    mesh's triangles and set-up time (ms, the icosphere's construction on the host included), and with mesh_scan
    the scan's statistics"""
    import numpy as np
    import torch
    from nksr_b200.training import TrainingScene
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    if kind == "sphere":
        from tests import clouds
        xyz, nrm = clouds.sphere(n, noise=0.001)
        W = 0.02 if n <= 300_000 else 0.01
        if not mesh_gt:
            return TrainingScene(t(xyz), t(nrm), W, depth), None
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        gt = build_mesh_gt(W, device)
        e1.record()
        torch.cuda.synchronize()
        info = dict(triangles=gt.mesh.n_tri, samples=int(gt.xyz.shape[0]), tau=gt.tau,
                    setup_ms=round(e0.elapsed_time(e1), 3))
        if not mesh_scan:
            return TrainingScene(t(xyz), t(nrm), W, depth, gt=gt), info
        px, pn, info["scan"] = scan_input(gt, n, device)
        return TrainingScene(px, pn, W, depth, gt=gt), info
    px, pn, ps, W = cfg4_crop(n, device)
    if not vol_sup:
        return TrainingScene(px, pn, W, depth), None
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    gt = build_volume(px, pn, ps, W, depth)
    e1.record()
    torch.cuda.synchronize()
    vol = dict(dims=list(gt.volume.shape), build_ms=round(e0.elapsed_time(e1), 3),
               fractions={k: round(v, 5) for k, v in gt.class_fractions().items()})
    return TrainingScene(px, pn, W, depth, gt=gt), vol


class KernelTimer:
    """CUDA events around every input-gradient (the forward kernel called from backward) and weight-gradient call"""

    def __init__(self, U):
        import torch
        self.U, self.phase, self.calls = U, "forward", []
        gemm, wgrad = U.gather_gemm, U.gather_gemm_wgrad

        def timed(kind, fn, shape):
            def run(*a, **k):
                if self.phase != "backward":
                    return fn(*a, **k)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = fn(*a, **k)
                e1.record()
                self.calls.append((kind, e0, e1, shape(*a)))
                return out
            return run
        U.gather_gemm = timed("dgrad", gemm, lambda x, idx, *r: None)
        U.gather_gemm_wgrad = timed("wgrad", wgrad, lambda x, idx, g, *r: (idx, x.shape[1], g.shape[1]))

    def summary(self):
        out = {"dgrad": 0.0, "wgrad": 0.0}
        for kind, e0, e1, _ in self.calls:
            out[kind] += e0.elapsed_time(e1)
        return out

    def wgrad_rates(self):
        """per (c_in, c_out): ms, TFLOP/s (2 nnz_taps c_in c_out) and GB/s (gathered x rows, g read once per tap with a
        source, the table, dW) of the weight-gradient kernel in the recorded step"""
        per = {}
        for kind, e0, e1, shp in self.calls:
            if kind != "wgrad":
                continue
            idx, ci, co = shp
            nnz = int((idx >= 0).sum())
            n_out, K = idx.shape
            r = per.setdefault(f"{ci}x{co}", dict(ms=0.0, flop=0.0, bytes=0.0, calls=0))
            r["ms"] += e0.elapsed_time(e1)
            r["flop"] += 2.0 * nnz * ci * co
            r["bytes"] += 4.0 * (nnz * ci + nnz * co + n_out * K + K * ci * co)
            r["calls"] += 1
        return {k: dict(ms=round(v["ms"], 3), calls=v["calls"], tflops=round(v["flop"] / v["ms"] / 1e9, 2),
                        gbs=round(v["bytes"] / v["ms"] / 1e6, 1)) for k, v in per.items()}


def structure_report(net, scene, pd, reps=5):
    """after training, without grad: per level the structure accuracy (argmax of the logits against the ground truth's
    voxel status on the hierarchy the decoder predicted for), |E_l|, |T_l| (the grown hierarchy) and |dec_l| (its kept
    voxels); the CUDA-event time of the growth step of every level; and the median forward time of the backbone
    (encoder hierarchy vs grown hierarchy under teacher forcing)"""
    import torch
    from nksr_b200 import structure as S
    from nksr_b200.svh import SparseIndexGrid
    D = min(net.backbone_net.depth, scene.enc_svh.depth)
    step_ms, orig = {}, S.StructureGrowth.step

    def timed_step(self, l, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        orig(self, l, *a, **k)
        e1.record()
        step_ms.setdefault(l, []).append((e0, e1))
    with torch.no_grad():
        enc = net.encoder(scene.xyz, scene.normal, scene.enc_svh, 0)
        gt = None if pd >= 1.0 else scene.gt_svh
        feat, dec, udf = net.unet(enc, scene.enc_svh, adaptive_depth=scene.adaptive_depth, gt_decoder_svh=gt)
        acc = {}
        for l, logits in feat.structure_features.items():
            if logits.shape[0]:
                want = scene.gt_svh.evaluate_voxel_status(SparseIndexGrid(udf, l), l)
                acc[l] = round(float((torch.argmax(logits, dim=1) == want).float().mean()), 4)
        sizes = [dict(level=l, enc=scene.enc_svh.num_voxels(l), grown=udf.num_voxels(l), dec=dec.num_voxels(l),
                      accuracy=acc.get(l)) for l in range(D)]
        times = {}
        S.StructureGrowth.step = timed_step
        try:
            for mode in ("encoder", "predicted"):
                grow = None if mode == "encoder" else dict(adaptive_depth=scene.adaptive_depth,
                                                          forced=S.teacher_classes(scene.gt_svh))
                ms = []
                for _ in range(reps):
                    step_ms.clear()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    net.backbone_net(enc.x0, scene.enc_svh, tf32=net.tf32, grow=grow)
                    e1.record()
                    torch.cuda.synchronize()
                    ms.append(e0.elapsed_time(e1))
                times[f"backbone_forward_{mode}_ms"] = round(statistics.median(ms), 3)
        finally:
            S.StructureGrowth.step = orig
        growth = {l: round(sum(a.elapsed_time(b) for a, b in v) / len(v), 3) for l, v in sorted(step_ms.items())}
    return dict(levels=sizes, growth_step_ms=growth, **times)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--scene", choices=("sphere", "cfg4"), default="sphere")
    ap.add_argument("--points", type=int, default=200_000)
    ap.add_argument("--depth", type=int, default=4)
    ap.add_argument("--precision", choices=("fp32", "tf32", "tc"), default="fp32")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="checkpoint path ({'state_dict': ...})")
    ap.add_argument("--kernel-losses", action="store_true", help="add the kernel-field losses (train through the solve)")
    ap.add_argument("--structure", choices=("encoder", "predicted"), default="encoder",
                    help="decoder hierarchy: the encoder's, or grown from the structure head (DESIGN.md SPEC S16)")
    ap.add_argument("--pd-structure-prob", type=float, default=0.0,
                    help="--structure predicted: probability of growing from the prediction instead of teacher forcing")
    ap.add_argument("--udf", action="store_true",
                    help="udf.enabled: the UDF loss on the NeuralField over every level (DESIGN.md SPEC S17)")
    ap.add_argument("--vol-sup", action="store_true",
                    help="cfg4: volume ground truth from the sensor rays (DESIGN.md SPEC S19)")
    ap.add_argument("--mesh-gt", action="store_true",
                    help="sphere: mesh ground truth, an icosphere of the scene's radius (DESIGN.md SPEC S21)")
    ap.add_argument("--mesh-scan", action="store_true",
                    help="--mesh-gt: the input is a simulated LiDAR scan of the mesh (DESIGN.md SPEC S22)")
    ap.add_argument("--operator", choices=("assembled", "matrix_free"), default=None,
                    help="--kernel-losses: the kernel solve's operator (default: assembled)")
    ap.add_argument("--geometry", choices=("kernel", "neural"), default="kernel",
                    help="output field: the kernel solve, or the NeuralField sdf_decoder(u(x)) (implies --kernel-losses)")
    args = ap.parse_args(argv)
    if args.geometry == "neural":
        args.kernel_losses = True
    if args.steps < 1:
        ap.error("--steps must be >= 1")
    if args.vol_sup and args.scene != "cfg4":
        ap.error("--vol-sup needs --scene cfg4 (its points carry their sensor positions)")
    if args.mesh_gt and args.scene != "sphere":
        ap.error("--mesh-gt needs --scene sphere (its ground-truth mesh is the icosphere of the same radius)")
    if args.mesh_scan and not args.mesh_gt:
        ap.error("--mesh-scan needs --mesh-gt (it scans the ground-truth mesh)")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("train_unet.py needs a CUDA device")
    import nksr_b200.unet as U
    from nksr_b200._lib import StageTimer
    from bench import gpu_info
    from nksr_b200 import training as T
    from nksr_b200.network import NKSRNetwork
    torch.use_deterministic_algorithms(True, warn_only=True)
    dev = torch.device("cuda:0")
    scene, vol = make_scene(args.scene, args.points, args.depth, dev, args.vol_sup, args.mesh_gt, args.mesh_scan)
    net = NKSRNetwork(dict(backbone="unet", tree_depth=args.depth, kernel_dim=4, precision=args.precision,
                           trainable=True, seed=args.seed, structure=args.structure,
                           udf=dict(enabled=args.udf), geometry=args.geometry)).to(dev)
    opt = T.make_optimizer(net)
    gen = torch.Generator(device=dev).manual_seed(args.seed)
    timer = KernelTimer(U)
    info = dict(gpu_info(0), scene=args.scene, points=int(scene.xyz.shape[0]), voxel_size=scene.voxel_size,
                depth=args.depth, precision=args.precision, structure=args.structure,
                pd_structure_prob=args.pd_structure_prob, udf=args.udf, geometry=args.geometry, operator=args.operator,
                voxels=[scene.enc_svh.num_voxels(l) for l in range(args.depth)])
    if vol is not None:
        info["mesh_gt" if args.mesh_gt else "volume"] = vol
    print(json.dumps(dict(setup=info)), flush=True)
    rows = []
    for step in range(args.steps):
        timer.calls.clear()
        ev = {"start": torch.cuda.Event(enable_timing=True)}
        ev["start"].record()

        def marks(name):
            ev[name] = torch.cuda.Event(enable_timing=True)
            ev[name].record()
            timer.phase = {"forward": "backward", "backward": "step"}.get(name, "forward")
        timer.phase = "forward"
        stages = StageTimer(dev, enabled=True) if args.kernel_losses else None
        out = T.train_step(net, opt, scene, gen, marks, kernel=args.kernel_losses, timer=stages,
                           pd_structure_prob=args.pd_structure_prob, operator=args.operator)
        l_struct, l_udf = out[:2]
        timer.phase = "forward"
        torch.cuda.synchronize()
        k = timer.summary()
        kern = {}
        if args.kernel_losses:
            st = stages.report()
            kern = {name: round(float(v), 6) for name, v in out[2].items()}
            kern.update(kernel_solve_ms=round(sum(st.get(s, 0.0) for s in ("kernel_rows", "gram_count", "gram_blocks",
                                                                           "gram_fill", "operator_setup", "pcg")), 3),
                        adjoint_pcg_ms=round(st.get("adjoint_pcg", 0.0), 3),
                        vjp_ms=round(st.get("feature_vjp", 0.0) + st.get("evaluate_vjp", 0.0), 3))
        row = dict(step=step, structure=round(float(l_struct), 6), udf=round(float(l_udf), 6), **kern,
                   forward_ms=round(ev["start"].elapsed_time(ev["forward"]), 3),
                   backward_ms=round(ev["forward"].elapsed_time(ev["backward"]), 3),
                   dgrad_ms=round(k["dgrad"], 3), wgrad_ms=round(k["wgrad"], 3),
                   step_ms=round(ev["backward"].elapsed_time(ev["step"]), 3))
        rows.append(row)
        print(json.dumps(row), flush=True)
    timed = rows[2:] if len(rows) > 2 else rows
    med = {key: round(statistics.median(r[key] for r in timed), 3)
           for key in ("forward_ms", "backward_ms", "dgrad_ms", "wgrad_ms", "step_ms", "kernel_solve_ms",
                       "adjoint_pcg_ms", "vjp_ms") if key in timed[0]}
    med["backward_over_forward"] = round(med["backward_ms"] / med["forward_ms"], 3)
    print(json.dumps(dict(summary=med, wgrad_last_step=timer.wgrad_rates(), **info)), flush=True)
    if args.structure == "predicted":
        print(json.dumps(dict(structure=structure_report(net, scene, args.pd_structure_prob))), flush=True)
    if args.out:
        torch.save({"state_dict": net.state_dict()}, args.out)


if __name__ == "__main__":
    main()
