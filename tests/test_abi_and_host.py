"""CPU-side checks: the C-ABI library loads and exports every symbol include/yolact_b200.h declares,
the host mirror reproduces the reference's state_dict keys, and the product path fails loudly
(no CPU fallback) when no GPU is present."""
import ctypes
import json
import os
import re

import pytest
import torch

import yolact_b200
from yolact_b200 import _lib
from yolact_b200.config import CONFIGS
from tests.conftest import GOLDEN, ROOT


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "yolact_b200.h")).read()
    return sorted(set(re.findall(r"^YB_API\s+[\w\s\*]+?\b(yb_[a-z0-9_]+)\s*\(", src, flags=re.M)))


def test_library_exports_every_declared_symbol():
    syms = _header_symbols()
    assert len(syms) >= 20
    assert os.path.exists(_lib.LIB_PATH), "build the library first: python -m yolact_b200.build"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in syms:
        assert hasattr(lib, s), "library does not export %s" % s
    # and the ctypes table covers exactly the header
    assert sorted(_lib.SIGNATURES) == syms
    assert _lib.load().yb_abi_version() == 2


def test_config_struct_matches_header_layout(tmp_path):
    # yb_config: 52 int32/float words (208 bytes, 8-byte aligned) followed by 24 doubles (ABI v2)
    n_words = 1 + 1 + 5 + 4 + 1 + 3 + 1 + 1 + 1 + 1 + 1 + 20 + 1 + 4 + 1 + 1 + 1 + 1 + 1 + 1 + 1
    assert ctypes.sizeof(_lib.YbConfig) == 4 * n_words + 8 * 24
    assert _lib.YbConfig.scales_f64.offset == 4 * n_words and _lib.YbConfig.ars_f64.offset == 4 * n_words + 8 * 20
    # the C compiler's view of the header must agree with the ctypes mirror
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "yolact_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu\\n", sizeof(yb_config), offsetof(yb_config, precision), '
                   'offsetof(yb_config, scales_f64), offsetof(yb_config, ars_f64)); return 0; }\n')
    exe = tmp_path / "layout"
    import subprocess
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [ctypes.sizeof(_lib.YbConfig), _lib.YbConfig.precision.offset, _lib.YbConfig.scales_f64.offset,
                   _lib.YbConfig.ars_f64.offset]


def test_conv_opts_struct_matches_header_layout(tmp_path):
    fields = ("cout_pad", "nseg", "seg_begin", "seg_pix_stride", "seg_batch_stride", "seg_y")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "yolact_b200.h"\n'
                   'int main(void) { printf("%zu' + ' %zu' * len(fields) + '\\n", sizeof(yb_conv_opts)' +
                   "".join(", offsetof(yb_conv_opts, %s)" % f for f in fields) + '); return 0; }\n')
    exe = tmp_path / "layout"
    import subprocess
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [ctypes.sizeof(_lib.YbConvOpts)] + [getattr(_lib.YbConvOpts, f).offset for f in fields]


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_state_dict_keys_match_reference(name):
    ref = json.load(open(os.path.join(GOLDEN, "state_keys.json")))[name]
    net = yolact_b200.Yolact(CONFIGS[name].copy())
    mine = {k: list(v.shape) for k, v in net.state_dict().items()}
    assert mine == ref


def test_set_cfg_and_side_effects():
    c = yolact_b200.set_cfg("yolact_im700_config")
    assert c.max_size == 700 and c.pred_scales == [[30], [61], [122], [244], [488]]   # config.py:721
    c = yolact_b200.set_cfg("yolact_plus_base")
    assert c.use_maskiou and not c.use_square_anchors and abs(c.pred_scales[0][1] - 30.238105197476955) < 1e-9
    yolact_b200.Yolact()
    assert yolact_b200.cfg.mask_dim == 32 and yolact_b200.cfg.num_heads == 5          # yolact.py:425,445
    yolact_b200.set_cfg("yolact_base_config")


def test_dcn_placement_rule():
    from yolact_b200.yolact import _block_uses_dcn
    # yolact_plus_base: [0,4,23,3], interval 3 -> every stage-first block + every 3rd block = 11 DCNs
    layers, dcn = [3, 4, 23, 3], [0, 4, 23, 3]
    n = sum(_block_uses_dcn(layers[i], dcn[i], 3, j) for i in range(4) for j in range(layers[i]))
    assert n == 11
    layers, dcn = [3, 4, 6, 3], [0, 4, 6, 3]
    n = sum(_block_uses_dcn(layers[i], dcn[i], 1, j) for i in range(4) for j in range(layers[i]))
    assert n == 13


def test_no_cpu_fallback():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    net = yolact_b200.Yolact(CONFIGS["yolact_resnet50_config"].copy())
    net.eval()
    with pytest.raises(_lib.YbError):
        net(torch.zeros(1, 3, 64, 64))
    # the C ABI itself refuses too
    lib = _lib.load()
    yc = _lib.YbConfig()
    yc.backbone = _lib.YB_BACKBONE_NONE
    yc.mask_dim = 32
    h = ctypes.c_void_p()
    assert lib.yb_create(ctypes.byref(yc), 0, ctypes.byref(h)) == -5   # YB_ERR_NO_DEVICE
    assert b"no CUDA device" in lib.yb_last_error()


def test_no_cpu_fallback_for_the_row_ops():
    """FastBaseTransform / mask_iou / jaccard / RLE / display blend: CPU tensors raise, nothing routes to torch ops."""
    from yolact_b200.augmentations import FastBaseTransform
    from yolact_b200 import eval_utils as E
    cfg = CONFIGS["yolact_base_config"].copy()
    with pytest.raises(_lib.YbError):
        FastBaseTransform(cfg)(torch.zeros(1, 8, 8, 3))
    m = torch.zeros(2, 4, 4)
    for call in (lambda: E.mask_iou(m, m), lambda: E.jaccard(torch.zeros(2, 4), torch.zeros(3, 4)),
                 lambda: E.encode_masks(m), lambda: E.pack_masks(m),
                 lambda: E.display_blend(torch.zeros(4, 4, 3), m, [[0, 0, 0]] * 2)):
        with pytest.raises(_lib.YbError):
            call()
    assert not hasattr(E, "prep_display")   # caller code (eval.py:135-262) is not rebuilt; only its blend is


def test_detect_nms_mode_follows_the_eval_flags():
    from yolact_b200.detection import Detect
    d = Detect(81, 0, 200, 0.05, 0.5)
    assert d.nms_mode() == _lib.YB_NMS_TRADITIONAL               # the reference class default (detection.py:30)
    d.use_fast_nms = True                                        # eval.py:871 with --fast_nms's default
    assert d.nms_mode() == _lib.YB_NMS_FAST
    d.second_threshold = True                                    # fast_nms(second_threshold=True), detection.py:160
    assert d.nms_mode() == (_lib.YB_NMS_FAST | _lib.YB_NMS_FLAG_SECOND_THRESHOLD)
    d.second_threshold = False
    d.use_cross_class_nms = True
    assert d.nms_mode() == _lib.YB_NMS_CROSS_CLASS
    d.use_fast_nms = False                                       # --fast_nms=False wins (detection.py:100-106)
    assert d.nms_mode() == _lib.YB_NMS_TRADITIONAL


def test_header_is_plain_c_and_links_from_c(tmp_path):
    """The boundary must be usable without C++ or torch: compile examples/c_abi_demo.c as C99 against the header,
    link it with the shared library only, run it."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    exe = str(tmp_path / "c_abi_demo")
    libdir = os.path.join(ROOT, "yolact_b200")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "c_abi_demo.c"), "-o", exe, os.path.join(libdir, "libyolact_b200.so"),
                    "-Wl,-rpath," + libdir], check=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    assert "yolact_b200 ABI 2" in out
    if not torch.cuda.is_available():
        assert "no CPU fallback" in out


def test_product_never_imports_oracle():
    for root, _, files in os.walk(os.path.join(ROOT, "yolact_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(root, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f


def test_graft_entry_build_check_passes():
    """The "does it build" entry point: (re)builds the library if a source is newer, loads it, checks the ABI
    version against the header and imports the oracle -- must hold on a machine without a GPU."""
    import __graft_entry__ as g
    assert g.build() is None
    src = open(os.path.join(ROOT, "include", "yolact_b200.h")).read()
    assert int(re.search(r"#define\s+YB_ABI_VERSION\s+(\d+)", src).group(1)) == _lib.ABI_VERSION == _lib.load().yb_abi_version()
