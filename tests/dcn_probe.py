"""Sampling-probe cases for the DCNv2 tests (host reference checks and the GPU edge tests share them).

A probe case is a DCNv2 call whose weights are a selection matrix: output channel o copies (tap t_o, input channel
c_o) with weight 1 and the bias is 0, so the output IS the im2col column and every sample is compared on its own.
The input is a ramp plus noise, so a sample taken from the wrong pixel is a large error.  The offsets of chosen
(pixel, tap) pairs are built so that the sampling position lands exactly (in fp32) on the places where the inside test,
the corner tests or the floor change their answer; all other pairs get Gaussian offsets.
"""
import numpy as np

f32 = np.float32
SEL_CHANNELS = 8          # selected input channels per tap -> Co = 72
MASK_VALUES = (1.0, 0.5, 1e-6, 1.0, 0.0)   # probe masks cycle through these; 1e-6 makes an fp16 weight subnormal
FAR_OFFSETS = (f32(-1e4), f32(1e4), f32(3e9), f32(-3e9), f32(np.nan), f32(np.inf), f32(-np.inf))


def out_hw(H, W, stride, pad, dil):
    return (H + 2 * pad - (2 * dil + 1)) // stride + 1, (W + 2 * pad - (2 * dil + 1)) // stride + 1


def axis_targets(n):
    """Positions along an axis of n pixels where a sampling decision changes: (name, fp32 position)."""
    return [("0", f32(0)), ("1", f32(1)), ("n-2", f32(n - 2)), ("n-1", f32(n - 1)),
            ("-1", f32(-1)), ("n", f32(n)),
            ("-1+ulp", np.nextafter(f32(-1), f32(0))), ("n-ulp", np.nextafter(f32(n), f32(0))),
            ("-0.5", f32(-0.5)), ("n-0.5", f32(n - 0.5))]


def axis_expectation(name, n):
    """What the reference's rules give along one axis at a named target: (pixel index, weight), or None when the
    position is outside.  (The two one-ulp-inside targets are left to the numeric references.)"""
    return {"0": (0, 1.0), "1": (1, 1.0), "n-2": (n - 2, 1.0), "n-1": (n - 1, 1.0), "-1": None, "n": None,
            "-0.5": (0, 0.5), "n-0.5": (n - 1, 0.5)}[name]


def _exact_bases(target, bases):
    """bases (integer grid positions before the offset) from which `target` is reached exactly in fp32."""
    off = (target - bases.astype(f32)).astype(f32)
    return (bases.astype(f32) + off).astype(f32) == target


def build_probe_case(H, W, stride, pad, dil, C, seed, B=None):
    r = np.random.RandomState(seed)
    Ho, Wo = out_hw(H, W, stride, pad, dil)
    if B is None:
        B = max(2, -(-600 // (Ho * Wo * 9)))
    th, tw = axis_targets(H), axis_targets(W)
    edge = [k for k in range(10) if k not in (1, 2)]           # the product in both axes leaves out 1 and n-2
    specs = [(("pos", k), None) for k in range(10)] + [(None, ("pos", k)) for k in range(10)]
    specs += [(("pos", a), ("pos", b)) for a in edge for b in edge]
    for k in range(len(FAR_OFFSETS)):
        specs += [(("far", k), None), (None, ("far", k)), (("far", k), ("far", (k + 3) % len(FAR_OFFSETS)))]

    taps = np.arange(9)
    base_h = (np.arange(Ho)[:, None] * stride - pad + (taps // 3)[None, :] * dil)   # [Ho, 9]
    base_w = (np.arange(Wo)[:, None] * stride - pad + (taps % 3)[None, :] * dil)    # [Wo, 9]
    offset = (r.standard_normal((B, 18, Ho, Wo)) * 1.5).astype(f32)
    mask = (1 / (1 + np.exp(-r.standard_normal((B, 9, Ho, Wo))))).astype(f32)
    pick = r.randint(0, 5, size=mask.shape)
    for v, val in enumerate((0.0, 1.0, 0.5, 1e-6)):           # pick == 4 keeps the sigmoid value
        mask[pick == v] = val
    used = np.zeros((B, Ho, Wo, 9), bool)
    probes = []
    for n, (sh, sw) in enumerate(specs):
        okh = np.ones((Ho, 9), bool) if sh is None or sh[0] == "far" else _exact_bases(th[sh[1]][1], base_h)
        okw = np.ones((Wo, 9), bool) if sw is None or sw[0] == "far" else _exact_bases(tw[sw[1]][1], base_w)
        free = np.argwhere(okh[None, :, None, :] & okw[None, None, :, :] & ~used)
        assert len(free), "no (pixel, tap) reaches %r exactly" % ((sh, sw),)
        b, ho, wo, t = free[r.randint(len(free))]
        used[b, ho, wo, t] = True
        p = {"b": int(b), "ho": int(ho), "wo": int(wo), "tap": int(t), "h": None, "w": None}
        for axis, spec, tg, base, ch in (("h", sh, th, base_h[ho, t], 2 * t), ("w", sw, tw, base_w[wo, t], 2 * t + 1)):
            if spec is None:
                continue
            if spec[0] == "pos":
                name, pos = tg[spec[1]]
                offset[b, ch, ho, wo] = f32(pos - f32(base))
                p[axis] = (name, pos)
            else:
                offset[b, ch, ho, wo] = FAR_OFFSETS[spec[1]]
                p[axis] = ("far", None)
        mask[b, t, ho, wo] = MASK_VALUES[n % len(MASK_VALUES)]
        probes.append(p)

    hh, ww = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    x = (0.5 * hh - 0.3 * ww)[None, None] + 0.17 * (np.arange(C) % 7)[None, :, None, None] \
        - 1.5 * np.arange(B)[:, None, None, None] + 0.05 * r.standard_normal((B, C, H, W))
    x = (x - x.mean()).astype(f32)
    sel_c = np.round(np.linspace(0, C - 1, SEL_CHANNELS)).astype(int)   # one channel in each 16-byte piece of 64
    weight = np.zeros((9 * SEL_CHANNELS, C, 3, 3), f32)
    sel = [(t, int(c)) for t in range(9) for c in sel_c]
    for o, (t, c) in enumerate(sel):
        weight[o, c, t // 3, t % 3] = 1
    return {"x": x, "offset": offset, "mask": mask, "weight": weight, "bias": np.zeros(len(sel), f32), "sel": sel,
            "sel_c": sel_c, "probes": probes, "stride": stride, "pad": pad, "dil": dil, "base_h": base_h,
            "base_w": base_w}


def selected_columns(cols, case):
    """columns [B,C,9,Ho,Wo] -> [B,72,Ho,Wo] in the order of the selection matrix's output channels."""
    return np.stack([cols[:, c, t] for t, c in case["sel"]], axis=1)


GEOMETRIES = [(s, pad, dil, H, W) for s in (1, 2) for pad, dil in ((1, 1), (2, 2), (0, 1)) for H, W in ((7, 5), (21, 19))]
