"""The persistent seq-128 attention backward (csrc/attention.cu) walks the (batch, head) items with a static stride
through two operand buffers per CTA (GPU).

B2_DEBUG_ATTN_CTAS caps the grid, so one CTA takes many items and switches buffers many times: ctx, lse, the keep bits
and d_qkv must be bitwise the same whatever the grid, and the fused QKV-bias sums (fp32 atomics in no fixed order)
the same to rounding.  The reference comparison of test_attention.py is run at config A's full size, where every CTA
of the default grid takes more than one item.
"""
import os

import pytest
import torch

from parity import padded_visibility
from test_attention import block_ids, check_against_reference, check_dbias, packed_layout, padded_masks, run

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
CAPS = (None, 1, 7, 131)


def run_capped(cap, *args, **kw):
    old = os.environ.pop("B2_DEBUG_ATTN_CTAS", None)
    try:
        if cap is not None:
            os.environ["B2_DEBUG_ATTN_CTAS"] = str(cap)
        return run(*args, **kw)
    finally:
        os.environ.pop("B2_DEBUG_ATTN_CTAS", None)
        if old is not None:
            os.environ["B2_DEBUG_ATTN_CTAS"] = old


def shapes():
    """(name, batch, heads): config A (384 items), one item above the default grid (1 CTA per SM), one below the SM
    count"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return [("config_a", 32, 12), ("grid_plus_1", sms + 1, 1), ("sms_minus_1", sms - 1, 1)]


def check_grid_independent(qkv, dctx, B, nh, p, **kw):
    base = run_capped(None, qkv, dctx, B, 128, nh, p, cache=True, dbias=True, **kw)
    for cap in CAPS[1:]:
        got = run_capped(cap, qkv, dctx, B, 128, nh, p, cache=True, dbias=True, **kw)
        for name, a, b in zip(("ctx", "lse", "d_qkv"), got[:3], base[:3]):
            assert torch.equal(a, b), (name, cap)
        if p > 0:
            assert torch.equal(got[4], base[4]), ("keep_bits", cap)
        bound = 1e-5 * base[2].double().abs().sum(0) + 1e-30
        assert bool(((got[3].double() - base[3].double()).abs() <= bound).all()), ("dbias", cap)
    check_dbias(base[3], base[2])


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("shape", range(3))
def test_padded_grid_independent(cuda_dev, shape, p):
    _, B, nh = shapes()[shape]
    torch.manual_seed(71 + shape)
    H = nh * 64
    mask = padded_masks(128, B, seed=shape)[:B].to(cuda_dev)
    qkv = torch.randn(B * 128, 3 * H, device=cuda_dev).to(bf)
    dctx = torch.randn(B * 128, H, device=cuda_dev).to(bf)
    check_grid_independent(qkv, dctx, B, nh, p, mask=mask)


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_packed_grid_independent(cuda_dev, p):
    torch.manual_seed(81)
    seg = packed_layout().to(cuda_dev)
    B, nh = seg.shape[0], 12
    H = nh * 64
    qkv = torch.randn(B * 128, 3 * H, device=cuda_dev).to(bf)
    dctx = torch.randn(B * 128, H, device=cuda_dev).to(bf)
    check_grid_independent(qkv, dctx, B, nh, p, seg=seg)


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_config_a_matches_reference(cuda_dev, p):
    """B = 32, S = 128, 12 heads: per (sequence, head) against HF's attention in float64"""
    torch.manual_seed(91)
    B, S, nh = 32, 128, 12
    H = nh * 64
    mask = padded_masks(S, B, seed=9)[:B].to(cuda_dev)
    qkv = torch.randn(B * S, 3 * H, device=cuda_dev).to(bf)
    dctx = torch.randn(B * S, H, device=cuda_dev).to(bf)
    out = run(qkv, dctx, B, S, nh, p, mask=mask, cache=True, dbias=True)
    vis = padded_visibility(mask, S)
    check_against_reference(qkv, dctx, vis, block_ids(vis), B, S, nh, p, out, 1)
    check_dbias(out[3], out[2])
