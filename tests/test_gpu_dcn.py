"""DCNv2 op-level drop-in (yolact_b200.dcn_v2) against the golden vectors and the oracle."""
import numpy as np
import pytest
import torch

from oracle import yolact_oracle as O
from tests.conftest import load_golden
from yolact_b200.dcn_v2 import dcn_v2_conv, DCN

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tag", ["s1", "s2"])
def test_dcn_forward_golden_f32(tag):
    g = load_golden("dcn_unit")
    t = lambda a: torch.from_numpy(a).cuda()
    s = int(g[tag + "_stride"])
    y = dcn_v2_conv(t(g[tag + "_x"]), t(g[tag + "_offset"]), t(g[tag + "_mask"]), t(g[tag + "_w"]), t(g[tag + "_bias"]),
                    s, 1, 1, 1).cpu().numpy()
    assert np.abs(y - g[tag + "_y"]).max() < 2e-5


def test_dcn_zero_offset_identity():
    # external/DCNv2/test.py:32-67: zero offsets, mask 0.5, identity kernel -> 2*out == input
    C = 16
    x = torch.randn(2, C, 12, 10, device="cuda")
    w = torch.zeros(C, C, 3, 3, device="cuda")
    w[torch.arange(C), torch.arange(C), 1, 1] = 1
    y = dcn_v2_conv(x, torch.zeros(2, 18, 12, 10, device="cuda"), torch.full((2, 9, 12, 10), 0.5, device="cuda"), w,
                    torch.zeros(C, device="cuda"), 1, 1, 1, 1)
    assert (2 * y - x).abs().max() < 1e-6


@pytest.mark.parametrize("C,stride", [(64, 1), (128, 2), (32, 1)])
def test_dcn_f16_paths_vs_oracle(C, stride):
    r = np.random.RandomState(C + stride)
    B, H, W, Co = 2, 21, 19, 96
    x = r.standard_normal((B, C, H, W)).astype(np.float32)
    w = (r.standard_normal((Co, C, 3, 3)) * (2.0 / (9 * C)) ** 0.5).astype(np.float32)
    bias = r.standard_normal(Co).astype(np.float32) * 0.1
    Ho, Wo = (H + 2 - 3) // stride + 1, (W + 2 - 3) // stride + 1
    off = (r.standard_normal((B, 18, Ho, Wo)) * 1.5).astype(np.float32)
    msk = (1 / (1 + np.exp(-r.standard_normal((B, 9, Ho, Wo))))).astype(np.float32)
    ref = O.dcn_v2_forward(x, off, msk, w, bias, stride, 1, 1)
    t = lambda a: torch.from_numpy(a).cuda()
    y = dcn_v2_conv(t(x), t(off), t(msk), t(w), t(bias), stride, 1, 1, 1, precision="f16tc").cpu().numpy()
    # C % 64 == 0 -> gather + tensor-core contraction; else the fused SIMT fp16 kernel.  fp16 operands.
    assert np.abs(y - ref).max() < 1e-2 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("C,stride", [(64, 1), (128, 2)])
def test_dcn_split_precision_vs_oracle(C, stride):
    """YB_PREC_F16X3: gather of hi+lo samples -> split columns -> three-pass tensor-core contraction; fp32-equivalent."""
    r = np.random.RandomState(7 * C + stride)
    B, H, W, Co = 2, 21, 19, 96
    x = r.standard_normal((B, C, H, W)).astype(np.float32)
    w = (r.standard_normal((Co, C, 3, 3)) * (2.0 / (9 * C)) ** 0.5).astype(np.float32)
    bias = r.standard_normal(Co).astype(np.float32) * 0.1
    Ho, Wo = (H + 2 - 3) // stride + 1, (W + 2 - 3) // stride + 1
    off = (r.standard_normal((B, 18, Ho, Wo)) * 1.5).astype(np.float32)
    msk = (1 / (1 + np.exp(-r.standard_normal((B, 9, Ho, Wo))))).astype(np.float32)
    ref = O.dcn_v2_forward(x, off, msk, w, bias, stride, 1, 1)
    t = lambda a: torch.from_numpy(a).cuda()
    y = dcn_v2_conv(t(x), t(off), t(msk), t(w), t(bias), stride, 1, 1, 1, precision="f16x3").cpu().numpy()
    assert np.abs(y - ref).max() < 2e-5 * max(1.0, np.abs(ref).max())


def test_dcn_module_names():
    m = DCN(64, 64, 3, 1, 1)
    assert sorted(k for k, _ in m.named_parameters()) == ["bias", "conv_offset_mask.bias", "conv_offset_mask.weight", "weight"]
