"""Route the reference's eval.py through the H100 path without editing a line of it (INTEGRATION.md section 1).

    import integration.use_b200 as ub
    ub.install("/path/to/yolact")          # BEFORE `import eval`
    import eval as E                        # the reference's eval.py, unchanged
    E.parse_args([...]); ... E.evaluate(net, dataset)

or, from the shell:   python -m integration.use_b200 /path/to/yolact --trained_model=... --benchmark

`install` puts the reference on sys.path, imports its modules and rebinds the names eval.py pulls from them
(`from yolact import Yolact`, `from layers.output_utils import postprocess`, `from utils.augmentations import
FastBaseTransform`, `from layers.box_utils import jaccard, mask_iou`) to this package's mirrors.  The reference `cfg`
stays the object eval.py mutates; it is snapshotted into yolact_b200.cfg each time a Yolact is constructed
(eval.py calls set_cfg before `Yolact()`, eval.py:1085-1097).
"""
import sys


def install(reference_root, mask_iou_on_gpu=True):
    if reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    import yolact_b200
    from yolact_b200 import eval_utils
    from yolact_b200.config import from_reference_cfg
    from yolact_b200.augmentations import FastBaseTransform as B200FastBaseTransform

    import data as ref_data                      # noqa: the reference's packages
    import yolact as ref_yolact
    import layers.output_utils as ref_output_utils
    import layers.box_utils as ref_box_utils
    import utils.augmentations as ref_aug

    class Yolact(yolact_b200.Yolact):
        """`Yolact()` with the reference's no-argument constructor: reads the reference's global cfg."""

        def __init__(self):
            yolact_b200.cfg.replace(from_reference_cfg(ref_data.cfg))
            super().__init__()

    class FastBaseTransform(B200FastBaseTransform):
        def __init__(self):
            super().__init__(from_reference_cfg(ref_data.cfg))

    # cfg keys the reference's callers flip on the GLOBAL cfg between calls (prep_display sets rescore_bbox = True around
    # postprocess, eval.py:147-151; --detect clears eval_mask_branch, eval.py:1074): the package snapshot would go stale,
    # so they are re-read from the live reference cfg on every postprocess call.
    live_keys = ("rescore_bbox", "rescore_mask", "eval_mask_branch", "mask_proto_debug")

    def postprocess(*args, **kwargs):
        for key in live_keys:
            if hasattr(ref_data.cfg, key):
                setattr(yolact_b200.cfg, key, getattr(ref_data.cfg, key))
        return yolact_b200.postprocess(*args, **kwargs)
    postprocess.__doc__ = yolact_b200.postprocess.__doc__

    ref_yolact.ReferenceYolact = ref_yolact.Yolact          # the PyTorch graph stays reachable
    ref_yolact.Yolact = Yolact
    ref_output_utils.postprocess = postprocess
    ref_aug.FastBaseTransform = FastBaseTransform
    if mask_iou_on_gpu:
        ref_box_utils.mask_iou = eval_utils.mask_iou
        ref_box_utils.jaccard = eval_utils.jaccard
    return {"Yolact": Yolact, "postprocess": postprocess, "FastBaseTransform": FastBaseTransform}


if __name__ == "__main__":
    import runpy
    root = sys.argv[1]
    install(root)
    sys.argv = [root + "/eval.py"] + sys.argv[2:]
    runpy.run_path(root + "/eval.py", run_name="__main__")   # the reference's eval.py, as its own __main__
