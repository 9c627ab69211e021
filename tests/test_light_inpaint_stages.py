"""CPU: the float64 stage references of light_inpaint_v1 (oracle/light_inpaint_stages.py), chained with their fp16 rounding
switched off, are the whole network: they equal oracle.light_inpaint in float64 and the reference's goldens
(tests/golden/light_inpaint.npz).  So a wrong decomposition cannot let the per-stage GPU tests
(tests/test_gpu_light_inpaint_stages.py) pass."""
import pytest
import torch

from tests.util import load_golden, t
from nunif_b200 import synth
from oracle import light_inpaint as oli
from oracle import light_inpaint_stages as ols


@pytest.fixture(scope="module")
def g():
    return load_golden("light_inpaint")


@pytest.fixture(scope="module")
def sd():
    return synth.light_inpaint_v1_state_dict(0)


def blur64(mask):
    """The blurred mask (oli.prepare_mask computes it in fp32) as float64, so that both sides composite in float64."""
    return oli.prepare_mask(mask, mask)[1].double()


def oracle64(sd, x, mask):
    return oli.network({k: v.double() for k, v in sd.items()}, x * (1 - mask), blur64(mask))


def chain(sd, x, mask, mirror):
    """The stage chain on the float64 inputs, the blur in network coordinates as the engine's tap 100 holds it."""
    return ols.forward(sd, x, mask, blur64(mask.flip(-1) if mirror else mask), mirror, r16=False)


@pytest.mark.parametrize("i", range(3))
def test_stage_chain_equals_oracle_network(g, sd, i):
    h, w = (int(v) for v in g[f"net{i}_hw"])
    x, mask = oli.net_inputs(int(g[f"net{i}_seed"]), 1, h, w)
    x, mask = x.double(), mask.double()
    with torch.no_grad():
        z = chain(sd, x, mask, 0)
        want = oracle64(sd, x, mask)
    assert z.dtype == torch.float64 and z.shape == want.shape
    assert (z - want).abs().max() <= 1e-9 * want.abs().max()
    # and the reference's own (fp32) output, with test_oracle_network_golden's tolerance
    assert (z - t(g[f"net{i}_z"]).double()).abs().max() <= 1e-5


def test_stage_chain_mirror(sd):
    """forward_left's mirror: the chain with mirror=1 is the network on the flipped frame and mask, flipped back."""
    x, mask = oli.net_inputs(21, 2, 70, 150)
    x, mask = x.double(), mask.double()
    with torch.no_grad():
        z = chain(sd, x, mask, 1)
        want = oracle64(sd, x.flip(-1), mask.flip(-1)).flip(-1)
    assert (z - want).abs().max() <= 1e-9 * want.abs().max()


def test_stage_shapes(sd):
    """Each stage's output has the shape of the engine tap that holds it (DESIGN.md §5)."""
    B, H, W = 2, 70, 150
    x, mask = oli.net_inputs(3, B, H, W)
    x, mask = x.double(), mask.double()
    _, blur = oli.prepare_mask(mask, x)
    Hp, Wp = ols.padded(H, W)
    assert (Hp, Wp) == (128, 192) and ols.padded(64, 256) == (128, 320)
    H4, W4 = Hp // 4, Wp // 4
    with torch.no_grad():
        x1, a1, tok = ols.stem(sd, x, mask, blur[:, 0], 0, r16=False)
        assert x1.shape == a1.shape == (B, H4, W4, 96) and tok.shape == (B, H4, W4)
        s = ols.block(sd, 0, x1, r16=False)
        assert [tuple(v.shape) for v in s] == [(B, H4, W4, 96), (B, H4 + 16, W4 + 16, 96), (B, H4 + 16, W4 + 16, 384),
                                               (B, H4 + 16, W4 + 16, 384), (B, H4, W4, 96), (B, H4, W4, 96),
                                               (B, H4 + 2, W4 + 2, 64), (B, H4, W4, 96)]
        x2 = ols.down(sd, s[-1], r16=False)[0]
        assert x2.shape == (B, H4 // 2, W4 // 2, 192)
        assert ols.block(sd, 1, x2, r16=False)[6].shape == (B, H4 // 2 + 2, W4 // 2 + 2, 96)
        assert ols.up(sd, x2, s[-1], r16=False)[0].shape == (B, H4, W4, 96)
