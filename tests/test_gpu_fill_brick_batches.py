"""The brick fill's batches (csrc/gram_fill_brick.cu): a block packs the consecutive bricks that start in its window of
64 voxel indices into batches of at most 64 rows and runs one phase schedule per batch.  Clouds built so that the
fine levels hold what only the batching can get wrong -- full 64-row bricks next to one-row bricks, batches cut by the
row capacity, a source voxel in the halo of two bricks of one batch, a voxel with hundreds of constraint locations --
each checked against the row fill and the oracle like the other brick tests."""
import numpy as np
import pytest

from tests import clouds
from tests.test_gpu_fill_brick import _compare, _hierarchy, _systems, every_level  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def _mixed_cloud(seed, dense_points=400):
    """a solid 8^3-voxel cube of points (full bricks on the finest levels), single points one and two voxels off its
    faces (bricks of one or a few rows beside it, sharing its halo), one voxel with `dense_points` points, and a
    sparse shell around all of it"""
    W = 0.02
    rng = np.random.default_rng(seed)
    g = (np.arange(8, dtype=np.float32) + 0.5) * W
    cube = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    side = np.array([[8.5, 3.5, 2.5], [9.5, 6.5, 0.5], [-0.5, 4.5, 4.5], [3.5, -1.5, 7.5], [2.5, 5.5, 9.5]],
                    np.float32) * W
    dense = (np.array([-5.5, 2.5, 1.5], np.float32) * W +
             rng.uniform(-0.3, 0.3, (dense_points, 3)).astype(np.float32) * W)
    shell, _ = clouds.shapenet_like(1500)
    return np.concatenate([cube, side, dense, shell]).astype(np.float32), W


def _brick_rows(osvh, l):
    _, counts = np.unique(np.asarray(osvh.keys[l]) >> 6, return_counts=True)
    return counts


@pytest.mark.parametrize("layout", ["levels", "interleaved"])
@pytest.mark.parametrize("prune", [0.0, 0.4])
def test_batches_mixed_bricks(cuda, every_level, layout, prune):
    xyz, W = _mixed_cloud(7)
    svh, osvh = _hierarchy(cuda, xyz, W, 4, prune, seed=3)
    rows0 = _brick_rows(osvh, 0)
    if prune == 0.0:
        assert rows0.max() == 64 and rows0.min() <= 4      # a full brick and small ones
    # bricks of consecutive rows that do not fit one batch together
    assert (rows0[:-1] + rows0[1:] > 64).any()
    out, ref = _systems(cuda, svh, osvh, xyz, W, False, 4, True, layout)
    worst = _compare(out, ref, osvh, f"mixed bricks prune={prune} {layout}")
    print(f"[brick batches] worst reorder ratios (values, diagonal, rhs): {worst}")


def test_batches_dense_voxel(cuda, every_level):
    """one voxel with 600 position constraints and its neighbours' normals: long location loops inside one item"""
    xyz, W = _mixed_cloud(8, dense_points=600)
    svh, osvh = _hierarchy(cuda, xyz, W, 3)
    out, ref = _systems(cuda, svh, osvh, xyz, W, True, 3, True, "levels")
    _compare(out, ref, osvh, "dense voxel")
