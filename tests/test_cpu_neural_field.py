"""NKSRNetwork's udf.enabled option (DESIGN.md SPEC S17): which backbones accept it, the width of the UDF decoder it
builds, and that it leaves every other parameter as it is with the option disabled."""
import pytest
import torch

from nksr_b200.network import NKSRNetwork


def test_pool_backbone_refuses_udf():
    with pytest.raises(ValueError, match="udf"):
        NKSRNetwork(dict(backbone="pool", udf=dict(enabled=True)))


@pytest.mark.parametrize("kernel_dim,tree_depth", [(4, 4), (8, 3)])
def test_unet_udf_decoder_reads_every_level_and_leaves_the_rest_unchanged(kernel_dim, tree_depth):
    hp = dict(backbone="unet", kernel_dim=kernel_dim, tree_depth=tree_depth, seed=3)
    on = NKSRNetwork(dict(hp, udf=dict(enabled=True)))
    off = NKSRNetwork(hp)
    dec = on.udf_decoder
    linears = [m for m in dec if isinstance(m, torch.nn.Linear)]
    assert [(m.in_features, m.out_features) for m in linears] == [(kernel_dim * tree_depth, 32), (32, 32), (32, 1)]
    assert [type(m) for m in dec] == [torch.nn.Linear, torch.nn.ReLU, torch.nn.Linear, torch.nn.ReLU, torch.nn.Linear]
    s_on, s_off = on.state_dict(), off.state_dict()
    others = [k for k in s_off if not k.startswith("udf_decoder.")]
    assert others == [k for k in s_on if not k.startswith("udf_decoder.")]
    for k in others:
        assert torch.equal(s_on[k], s_off[k]), k
    # the UDF decoder's own seed: the same for the same network seed, different for another
    again = NKSRNetwork(dict(hp, udf=dict(enabled=True)))
    assert all(torch.equal(a, b) for a, b in zip(dec.parameters(), again.udf_decoder.parameters()))
    other = NKSRNetwork(dict(hp, seed=4, udf=dict(enabled=True)))
    assert not torch.equal(linears[0].weight, other.udf_decoder[0].weight)
    # the global random stream is left as it was
    torch.manual_seed(11)
    a = torch.rand(4)
    torch.manual_seed(11)
    NKSRNetwork(dict(hp, udf=dict(enabled=True)))
    assert torch.equal(torch.rand(4), a)


@pytest.mark.parametrize("backbone", ["pool", "unet"])
def test_udf_disabled_keeps_the_single_level_decoder(backbone):
    net = NKSRNetwork(dict(backbone=backbone, kernel_dim=4, tree_depth=4))
    assert not net.udf_enabled
    first = net.udf_decoder[0]
    assert isinstance(first, torch.nn.Linear) and (first.in_features, first.out_features) == (4, 16)
    assert [k for k in net.state_dict() if k.startswith("udf_decoder.")] == [
        "udf_decoder.0.weight", "udf_decoder.0.bias", "udf_decoder.2.weight", "udf_decoder.2.bias"]
