"""Fused attention at the edges of its 16-row query / key tiles and on both sides of the split of an (image, head)
pair over several CTAs (attn_plan_make splits a pair's tiles when there are fewer pairs than SMs), against the float64
reference and per-element budgets of test_attn_gpu.py.  _run's guard bands catch any write past the tensors."""
import pytest

from test_attn_gpu import _case, _inputs

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("T", [15, 16, 17, 31, 33, 47, 49, 79, 81, 111, 113, 207, 208, 209, 223, 225])
@pytest.mark.parametrize("B,H", [(1, 1), (3, 12)])
def test_attention_tile_edges(T, B, H):
    qkv, d_o = _inputs(B, T, H, 11 * T + B + H)
    _case(f"tile edges B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)


# one pair split over 13 CTAs; 96 pairs, two CTAs each on a 132-SM H100; 768 pairs, one CTA each
@pytest.mark.parametrize("B,H", [(1, 1), (8, 12), (64, 12)])
def test_attention_pair_split(B, H):
    T = 197
    qkv, d_o = _inputs(B, T, H, 17 * B + H)
    _case(f"pair split B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)
