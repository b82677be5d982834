"""The size-dependent tables of every image geometry the GPU tests run (tests/stages.py GEOMETRIES) and of the golden
fixtures, against the oracle, on the CPU: the interpolated position embedding, the padded sine table of the head
transformers, the N x N row pitch and the sampler's load mode that pitch selects."""
import pytest
import torch

from mickey_b200.engine import interpolate_pos_embed, nn_pitch, sine_table_padded
from oracle import mickey_oracle as mo
from tests import stages as st
from tests.common import GOLDEN_CASES

SIZES = {**{k: (v[2], v[3]) for k, v in st.GEOMETRIES.items()},
         **{k: (v["height"], v["width"]) for k, v in GOLDEN_CASES.items()}}


@pytest.mark.parametrize("name", sorted(SIZES))
def test_interpolate_pos_embed_is_the_oracle(name):
    H, W = SIZES[name]
    gh, gw = H // 14, W // 14
    pos = torch.randn(1, 1 + 37 * 37, 384, generator=torch.Generator().manual_seed(gh * 100 + gw))
    got = interpolate_pos_embed(pos, gh, gw)
    ref = mo.interpolate_pos_embed(pos, gh, gw)[0]
    assert got.shape == (1 + gh * gw, 384) and torch.equal(got, ref)
    assert torch.equal(got[0], pos[0, 0])
    if (gh, gw) == (37, 37):                         # the identity branch: no resize at all
        assert torch.equal(got, pos[0])
    else:
        assert not torch.equal(got[1:38], pos[0, 1:38])


@pytest.mark.parametrize("name", sorted(SIZES))
def test_sine_table_padded_is_the_oracle(name):
    H, W = SIZES[name]
    gh, gw = H // 14, W // 14
    got = sine_table_padded(gh, gw).reshape(gh + 2, gw + 2, 128)
    ref = mo.sine_position_encoding(128, gh, gw).permute(1, 2, 0)
    assert torch.equal(got[1:-1, 1:-1], ref)
    ring = got.clone()
    ring[1:-1, 1:-1] = 0
    assert float(ring.abs().max()) == 0.0


@pytest.mark.parametrize("name", sorted(st.GEOMETRIES))
def test_pitch_and_sampler_mode(name, monkeypatch):
    monkeypatch.setenv("MICKEY_NN_CONTIGUOUS", "1")           # has no effect: the engine's N x N pitch is always padded
    _, _, H, W, _, _, _ = st.GEOMETRIES[name]
    (gh, gw), N, pitch, mode = st.GEOMETRY_PATHS[name]
    assert (H // 14, W // 14) == (gh, gw) and gh * gw == N
    assert nn_pitch(N) == pitch
    assert st.sampler_mode(N, pitch) == mode
    assert st.sampler_mode(N, N) == ("FLAT_VEC" if N * N % 4 == 0 else "SCALAR")       # caller tensors at pitch N
    assert st.sampler_mode(N, pitch, aligned=False) == "SCALAR"


def test_geometries_reach_their_paths():
    """What each GPU run is there for, from its numbers."""
    g = {k: st.GEOMETRY_PATHS[k] for k in st.GEOMETRIES}
    T = {k: v[1] + 1 for k, v in g.items()}
    assert g["land"][0][1] > g["land"][0][0] and g["land"][1] == 1938
    assert g["n1920"][1] % 128 == 0 and T["n1920"] % 192 == 1
    assert T["t2304"] % 192 == 0 and T["t2304"] % 128 == 0 and (2 * T["t2304"]) % 128 == 0 and g["t2304"][1] % 2 == 1
    _, _, H, W, _, _, _ = st.GEOMETRIES["crop"]
    assert H % 14 == 13 and W % 14 == 13
    assert g["min"][0] == (7, 7) and (g["min"][0][0] - 6) * (g["min"][0][1] - 6) == 1 and 2 * T["min"] < 128
    assert g["sq37"][0] == (37, 37)
    assert g["large"][1] > 4097
