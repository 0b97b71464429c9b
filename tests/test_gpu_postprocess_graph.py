"""The dense postprocess calls (assemble_masks, assemble_masks_batch) upload nothing and synchronise nothing, so a
caller can capture them into a CUDA graph: replaying the graph must give what eager calls give, for the inputs the
graph's tensors hold at replay time.  Also: a mask launch whose shared-memory tables only pass 48 KB with the
kernel's static shared memory added still runs."""
import numpy as np
import pytest
import torch

from yolact_b200.output_utils import assemble_masks, assemble_masks_batch

pytestmark = pytest.mark.gpu


def inputs(B, n, ph, pw, k, seed):
    r = np.random.RandomState(seed)
    proto = np.maximum(r.standard_normal((B, ph, pw, k)), 0).astype(np.float32)
    coef = np.tanh(r.standard_normal((B, n, k))).astype(np.float32)
    c, wh = r.uniform(0.2, 0.8, (B, n, 2)), r.uniform(0.05, 0.6, (B, n, 2))
    box = np.concatenate([c - wh / 2, c + wh / 2], 2).astype(np.float32)
    return [torch.from_numpy(a).cuda() for a in (proto, coef, box)]


@pytest.mark.parametrize("fmt", ["f32", "u8", "bits"])
def test_dense_postprocess_replays_from_a_cuda_graph(fmt):
    B, n, h, w = 3, 17, 101, 135
    proto, coef, box = inputs(B, n, 40, 44, 32, 7)

    def run():
        return (assemble_masks_batch(proto, coef, box, h, w, True, fmt),
                assemble_masks(proto[1], coef[1], box[1], h, w, True, fmt, want_proto_masks=True))

    run()   # creates the ops handle and sets the kernels' shared-memory attributes outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        captured = run()
    for step in range(2):
        if step:
            coef.neg_()          # the graph reads its inputs when it is replayed
            box.mul_(0.9)
        g.replay()
        eager = run()
        torch.cuda.synchronize()
        (gm, gb), (gm1, gb1, gp1) = captured
        (em, eb), (em1, eb1, ep1) = eager
        assert torch.equal(gm, em) and torch.equal(gb, eb), (fmt, step)
        assert torch.equal(gm1, em1) and torch.equal(gb1, eb1) and torch.equal(gp1, ep1), (fmt, step)
        assert int(em.count_nonzero()) > 0 and int(ep1.count_nonzero()) > 0, (fmt, step)


def test_mask_tables_just_under_48_kb_launch_in_a_fresh_process():
    """At 720x2896 from 138x138 prototypes the mask kernel's dynamic shared memory is 49096 bytes: under 48 KB, but not
    once its static shared memory is added, so the launch must opt in to more.  A fresh process has not opted in yet."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = """
import sys
sys.path.insert(0, %r)
import torch
from tests.test_gpu_postprocess_graph import inputs
from yolact_b200.output_utils import assemble_masks, unpack_bits
proto, coef, box = inputs(1, 9, 138, 138, 32, 3)
m = {f: assemble_masks(proto[0], coef[0], box[0], 720, 2896, True, f)[0] for f in ('u8', 'f32', 'bits')}
assert torch.equal(m['u8'], m['f32'].to(torch.uint8)) and torch.equal(m['u8'], unpack_bits(m['bits'], 2896))
assert int(m['u8'].count_nonzero()) > 0
print('ok')
""" % root
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stdout + r.stderr
