"""Multi-GPU check of nksr_b200/dist_solve.py (run under torchrun, one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tools/check_global_solve.py \
        [--operator assembled|matrix_free]

Every rank builds the same seeded elongated cloud; the ranks solve ONE global system sharded by
slabs (halo exchange + all-reduced dot products), rank 0 additionally solves the same system alone,
and the coefficients are compared unknown by unknown through their (level, Morton key)."""
import argparse
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nksr_b200  # noqa: E402
from nksr_b200 import dist_solve as ds  # noqa: E402


def capsule(n, length=12.0, radius=0.5, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-length / 2, length / 2, n)
    th = rng.uniform(0, 2 * np.pi, n)
    nrm = np.stack([np.zeros(n), np.cos(th), np.sin(th)], 1)
    xyz = np.stack([x, radius * np.cos(th), radius * np.sin(th)], 1) + rng.normal(size=(n, 3)) * 0.002
    return xyz.astype(np.float32), nrm.astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--operator", choices=("assembled", "matrix_free"), default=None,
                    help="the global solve's operator (default: NKSR_OPERATOR, else assembled)")
    args = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    solo = dist.new_group([0])
    xyz, nrm = capsule(200_000)
    W = 0.05
    rec = nksr_b200.Reconstructor(dev, tree_depth=3)
    t = lambda a: torch.from_numpy(a).to(dev)
    field = ds.reconstruct_global(rec, t(xyz), t(nrm), W, halo_voxels=8, solver_tol=1e-6, operator=args.operator)
    info = field.solve_info
    mesh = ds.extract_global_mesh(field, mise_iter=1)
    # owned coefficients with their (level, key) identity
    offs = field.svh.offsets
    lv = torch.cat([torch.full((field.svh.num_voxels(l),), l, dtype=torch.int64, device=dev) for l in range(3)])
    keys = torch.cat(field.svh.keys)
    own = field.owned
    mine = (lv[own].cpu().numpy(), keys[own].cpu().numpy(), field.alpha[own].cpu().numpy())
    gathered = [None] * world
    dist.all_gather_object(gathered, (mine, info))
    ok = True
    if rank == 0:
        ref = ds.reconstruct_global(rec, t(xyz), t(nrm), W, halo_voxels=8, solver_tol=1e-6, group=solo,
                                    operator=args.operator)
        rk = torch.cat(ref.svh.keys).cpu().numpy()
        rl = np.concatenate([np.full(ref.svh.num_voxels(l), l) for l in range(3)])
        ra = ref.alpha.cpu().numpy()
        lut = {(int(l), int(k)): float(a) for l, k, a in zip(rl, rk, ra)}
        total, worst, scale = 0, 0.0, float(np.abs(ra).max())
        for r, ((l_, k_, a_), inf) in enumerate(gathered):
            total += len(a_)
            d = np.array([abs(lut[(int(l), int(k))] - float(a)) for l, k, a in zip(l_, k_, a_)])
            worst = max(worst, float(d.max()))
            print(f"rank {r}: owned {len(a_)} of local {inf['n']} unknowns, halo {inf['halo_recv']}, iters {inf['iterations']}, "
                  f"relres {inf['relative_residual']:.2e}, operator {inf['operator']}, kept locations "
                  f"{inf.get('locations_kept')} of {inf.get('locations_total')}, slab {inf['slab']}, max |alpha - ref| = {d.max():.3e}")
        ok &= total == len(ra)                      # every unknown owned exactly once
        ok &= worst <= 2e-3 * scale
        refmesh = ref.extract_dual_mesh(mise_iter=1)
        rr = np.linalg.norm(mesh.v.cpu().numpy()[:, 1:], axis=1)
        print(f"unknowns {len(ra)} (union of owned {total}); ref iters {ref.solve_info['iterations']}; "
              f"worst/scale = {worst / scale:.2e}; mesh faces {mesh.f.shape[0]} vs single {refmesh.f.shape[0]}; "
              f"radius median {np.median(rr):.4f}")
        ok &= abs(mesh.f.shape[0] - refmesh.f.shape[0]) <= 0.01 * refmesh.f.shape[0] + 16
        ok &= abs(np.median(rr) - 0.5) < 0.01
        print("GLOBAL-SOLVE CHECK", "PASS" if ok else "FAIL")
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
