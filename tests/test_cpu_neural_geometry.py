"""NKSRNetwork's geometry option (models/nksr_net.py:89-122): which values and backbones it accepts, the SDF decoder
geometry='neural' builds and that every other parameter stays what it is with 'kernel'; and the fp64 restatement of the
neural field's position Jacobian (tests/jacobian_oracle.py, DESIGN.md SPEC S17a) against central finite differences of
the fp64 interpolation."""
import numpy as np
import pytest
import torch

from nksr_b200.network import NKSRNetwork
from oracle import nksr_oracle as O
from tests import clouds
from tests.jacobian_oracle import interp64, jacobian64


def test_geometry_values_and_backbones():
    assert NKSRNetwork().geometry == "kernel"
    with pytest.raises(ValueError, match="geometry"):
        NKSRNetwork(dict(backbone="unet", geometry="implicit"))
    with pytest.raises(ValueError, match="geometry='neural' needs backbone='unet'"):
        NKSRNetwork(dict(backbone="pool", geometry="neural"))


@pytest.mark.parametrize("kernel_dim,tree_depth,udf", [(4, 4, False), (8, 3, True)])
def test_neural_sdf_decoder_reads_every_level_and_leaves_the_rest_unchanged(kernel_dim, tree_depth, udf):
    hp = dict(backbone="unet", kernel_dim=kernel_dim, tree_depth=tree_depth, seed=3, udf=dict(enabled=udf))
    on = NKSRNetwork(dict(hp, geometry="neural"))
    off = NKSRNetwork(dict(hp, geometry="kernel"))
    dec = on.sdf_decoder
    linears = [m for m in dec if isinstance(m, torch.nn.Linear)]
    assert [(m.in_features, m.out_features) for m in linears] == [(kernel_dim * tree_depth, 32), (32, 32), (32, 1)]
    assert [type(m) for m in dec] == [torch.nn.Linear, torch.nn.ReLU, torch.nn.Linear, torch.nn.ReLU, torch.nn.Linear]
    s_on, s_off = on.state_dict(), off.state_dict()
    others = [k for k in s_off if not k.startswith("sdf_decoder.")]
    assert others == [k for k in s_on if not k.startswith("sdf_decoder.")]
    for k in others:
        assert torch.equal(s_on[k], s_off[k]), k
    # the SDF decoder's own seed: the same for the same network seed, different for another, and not the UDF decoder's
    again = NKSRNetwork(dict(hp, geometry="neural"))
    assert all(torch.equal(a, b) for a, b in zip(dec.parameters(), again.sdf_decoder.parameters()))
    other = NKSRNetwork(dict(hp, seed=4, geometry="neural"))
    assert not torch.equal(linears[0].weight, other.sdf_decoder[0].weight)
    if udf:
        assert not torch.equal(linears[0].weight, on.udf_decoder[0].weight)
    # the global random stream is left as it was
    torch.manual_seed(11)
    a = torch.rand(4)
    torch.manual_seed(11)
    NKSRNetwork(dict(hp, geometry="neural"))
    assert torch.equal(torch.rand(4), a)


@pytest.mark.parametrize("depth,W", [(1, 0.05), (3, 0.05), (4, 0.05)])
def test_jacobian_oracle_against_finite_differences(depth, W):
    xyz, _ = clouds.sphere(3000, noise=0.001)
    osvh = O.OracleSVH(W, depth).build_point_splatting(xyz)
    rng = np.random.default_rng(depth)
    C = 3
    feats = {l: rng.normal(size=(osvh.n(l), C)) for l in range(depth)}
    levels = list(range(depth))
    q = np.concatenate([xyz[:800], xyz[:800] + rng.normal(0.0, 0.02, (800, 3))]).astype(np.float64)
    h = 1.0e-3 * W
    # away from voxel centres (|tau| > 0.01 on every level), and with x -+ h e_a in the same voxels as x on every level:
    # there u is linear along each axis, so the central difference is exact up to rounding
    keep = np.ones(q.shape[0], bool)
    base = osvh.locate(q)
    for l in range(depth):
        _, tau = O._level_tau(osvh, l, q, base[l])
        keep &= (base[l] < 0) | (np.abs(tau) > 0.01).all(axis=1)
    for a in range(3):
        e = np.zeros(3)
        e[a] = h
        keep &= (osvh.locate(q + e) == base).all(axis=0) & (osvh.locate(q - e) == base).all(axis=0)
    q = q[keep]
    assert q.shape[0] > 1000
    J, scale = jacobian64(osvh, feats, levels, q)
    assert (J != 0).any()
    for a in range(3):
        e = np.zeros(3)
        e[a] = h
        fd = (interp64(osvh, feats, levels, q + e) - interp64(osvh, feats, levels, q - e)) / (2 * h)
        np.testing.assert_allclose(J[:, a], fd, rtol=0, atol=1e-8 * (float(scale.max()) + 1.0))
    # outside every voxel: zero rows
    far = np.array([[5.0, 5.0, 5.0], [-4.0, 0.0, 0.0]])
    Jf, _ = jacobian64(osvh, feats, levels, far)
    assert not Jf.any()
