"""render_masks' argument checks, which run before anything touches a GPU."""
import pytest
import torch

from yolact_b200 import _lib
from yolact_b200.display import render_masks


def _det():
    return {"detection": {"box": torch.zeros(2, 4), "mask": torch.zeros(2, 32), "class": torch.zeros(2, dtype=torch.long),
                          "score": torch.ones(2), "proto": torch.zeros(8, 8, 32)}, "net": None}


def test_render_masks_has_no_cpu_path():
    with pytest.raises(_lib.YbError):
        render_masks([_det()], [torch.zeros(8, 8, 3, dtype=torch.uint8)])


def test_render_masks_needs_one_frame_per_detection():
    with pytest.raises(ValueError, match="2 frames for 1"):
        render_masks([_det()], [torch.zeros(8, 8, 3, dtype=torch.uint8)] * 2)
    with pytest.raises(ValueError, match="1 frames for 2"):
        render_masks([_det(), _det()], torch.zeros(1, 8, 8, 3, dtype=torch.uint8))
