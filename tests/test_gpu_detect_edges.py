"""Detect (csrc/detect.cu) decision by decision at its edges, against the reference's golden
(tests/golden/detect_edges.npz) and, where the golden is too small, against the oracle that
tests/test_detect_edges_oracle.py pins to it:

  * parameters: C = 2 (empty fg-max loop) / 21 / 96 / 97 / 129, top_k = 1 / 7 / 256, max_dets = 1 / 100, nms_thresh
    0.3 / 0.5 / 0.7, conf_thresh 0.05 / 0.5, a batch whose middle image has no candidate;
  * selection: M = top_k - 1 / top_k / top_k + 1, equal scores, a tie group across the cut, scores one ulp apart, key
    sets whose cut is decided by each radix pass, the traditional walk's 256-key chunk boundary, P around K1's tile;
  * thresholds: probabilities exactly float32(conf_thresh) and the next float up, box pairs whose IoU is exactly
    float32(nms_thresh) and pairs within a few ulp of it, with a float64 audit that the fixtures sit close enough to
    their thresholds for an FMA-contracted decode_box / box_iou to change a decision;
  * NaN probabilities, logits and boxes; parameter sets the launcher must refuse.

Exactness: counts, class ids, scores and coefficients bit for bit; boxes bit for bit where loc[:, 2:] == 0 (expf(0) = 1
and the decode is then round-to-nearest only), within 2 ulp of the row's largest coordinate elsewhere (expf).  Every
output starts as NaN; rows past the count must come back exactly zero.  The C ABI takes mask_dim in multiples of 4, so
the golden's mask_dim 1 and 33 run as 4 and 36 with the extra coefficient columns checked like the others.
"""
import numpy as np
import pytest
import torch

from oracle import yolact_oracle as O
from tests.conftest import load_golden
from tests.error_bounds import U24
from tests.test_detect_edges_oracle import assert_box_ulps
from yolact_b200 import _lib
from yolact_b200.detection import Detect

pytestmark = pytest.mark.gpu

MODES = ("fast", "cc", "trad")
_DETECTS = {}
SOFTMAX_RATIO = []


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if SOFTMAX_RATIO:
        print("largest |score - softmax64| / (softmax64 (C + 2) 2^-24): %.3f" % max(SOFTMAX_RATIO))


def detector(C, mode, top_k=200, max_dets=100, nms=0.5, conf_thresh=0.05, max_size=550):
    key = (C, mode, top_k, max_dets, nms, conf_thresh, max_size)
    if key not in _DETECTS:
        d = Detect(C, 0, top_k, conf_thresh, nms)
        d.use_fast_nms, d.use_cross_class_nms = mode != "trad", mode == "cc"
        d.max_num_detections, d.max_size = max_dets, max_size
        _DETECTS[key] = d
    return _DETECTS[key]


def run(d, loc, conf, mask, priors, logits=False, max_out=None, flags=0):
    """yb_detect with every output filled with NaN (class ids with -7) first.  Returns numpy (box, coef, cls, score,
    count) and the number of kernel launches.  flags: extra mode bits, for combinations Detect does not build."""
    lib = _lib.load()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    loc, conf, mask, priors = t(loc), t(conf), t(mask), t(priors)
    d.mask_dim = int(mask.shape[-1])      # the handle's mask_dim is the coefficient row stride
    h = d._handle(loc.device)
    B, P = int(loc.shape[0]), int(priors.shape[0])
    mode = d.nms_mode() | flags
    M = max_out if max_out is not None else (d.top_k if (mode & 0xFF) == _lib.YB_NMS_CROSS_CLASS else
                                             d.max_num_detections)
    nan = float("nan")
    box = torch.full((B, M, 4), nan, device="cuda")
    coef = torch.full((B, M, mask.shape[-1]), nan, device="cuda")
    cls = torch.full((B, M), -7, dtype=torch.int64, device="cuda")
    score = torch.full((B, M), nan, device="cuda")
    count = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    n0 = lib.yb_launch_count(h)
    _lib.check(lib.yb_detect(h, _lib.ptr(loc), _lib.ptr(conf), _lib.ptr(mask), _lib.ptr(priors), B, P,
                             1 if logits else 0, mode, M, _lib.ptr(box), _lib.ptr(coef), _lib.ptr(cls), _lib.ptr(score),
                             _lib.ptr(count), _lib.current_stream()), "yb_detect")
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in (box, coef, cls, score, count)], lib.yb_launch_count(h) - n0


def oracle(loc, conf, mask, priors, mode, top_k=200, max_dets=100, nms=0.5, conf_thresh=0.05, max_size=550):
    with np.errstate(invalid="ignore"):
        return O.detect_one(loc, conf, mask, priors, conf_thresh=conf_thresh, nms_thresh=nms, top_k=top_k,
                            max_dets=max_dets, cross_class=mode == "cc", traditional=mode == "trad", max_size=max_size)


def prior_of(coef):
    """The prior behind each output row, from its last coefficient column (see with_index_column)."""
    return coef[:, -1].astype(np.int64) if coef.shape[0] else np.zeros(0, np.int64)


def with_index_column(mask):
    """mask plus a last column holding the prior index, padded to a multiple of 4 columns (the ABI's mask_dim)."""
    B, P, K = mask.shape
    Kp = (K + 1 + 3) // 4 * 4
    out = np.zeros((B, P, Kp), np.float32)
    out[..., :K] = mask
    out[..., Kp - 1] = np.arange(P, dtype=np.float32)
    return out


def check_image(got, b, want, loc):
    """One image of a detect call against a reference result dict (or None), by the module's exactness rules."""
    box, coef, cls, score, count = got
    n = 0 if want is None else want["score"].shape[0]
    assert int(count[b]) == n
    M = box.shape[1]
    # rows past the count: exactly zero in every output
    assert (box[b, n:] == 0).all() and (coef[b, n:] == 0).all() and (cls[b, n:] == 0).all() and (score[b, n:] == 0).all()
    if n == 0:
        return
    assert n <= M
    assert np.array_equal(cls[b, :n], want["class"])
    assert np.array_equal(score[b, :n], want["score"])
    K = want["mask"].shape[1]
    assert np.array_equal(coef[b, :n, :K], want["mask"])
    pr = prior_of(coef[b, :n])
    exact = np.all(loc[pr][:, 2:] == 0, axis=1)
    assert np.array_equal(box[b, :n][exact], want["box"][exact], equal_nan=True)
    assert np.array_equal(np.isnan(box[b, :n]), np.isnan(want["box"]))
    assert_box_ulps(box[b, :n], want["box"], b)


def check_call(d, loc, conf, mask, priors, wants, mode, logits=False):
    """Poisoned outputs, three identical calls, each image equal to its single-image call, the launch count."""
    m = with_index_column(mask)
    got, launches = run(d, loc, conf, m, priors, logits)
    assert launches == (2 if mode == "cc" else 3)
    for _ in range(2):       # K1's atomic compaction order varies between runs; the result may not
        again, _ = run(d, loc, conf, m, priors, logits)
        for x, y in zip(got, again):
            assert np.array_equal(x, y, equal_nan=True)
    for b in range(loc.shape[0]):
        check_image(got, b, wants[b], loc[b])
        if loc.shape[0] > 1:
            one, _ = run(d, loc[b:b + 1], conf[b:b + 1], m[b:b + 1], priors, logits)
            for x, y in zip(got, one):
                assert np.array_equal(x[b], y[0], equal_nan=True)
    return got


# ---------------------------------------------------------------------------------------------------------------------
# the reference's own results
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def g():
    return load_golden("detect_edges")


def golden_wants(g, tag, B, K):
    out = []
    for b in range(B):
        if int(g[tag + "_counts"][b]) == 0:
            out.append(None)
        else:
            out.append({k: g["%s_%d_%s" % (tag, b, k)] for k in ("box", "mask", "class", "score")})
            assert out[-1]["mask"].shape[1] == K
    return out


@pytest.mark.parametrize("C", [2, 21, 96, 129])
def test_golden_edges(g, C):
    loc, conf, mask, priors = (g["C%d_%s" % (C, k)] for k in ("loc", "conf", "mask", "priors"))
    for i, row in enumerate(g["cases"]):
        if int(row[0]) != C:
            continue
        _, mode, top_k, max_dets, nms, conf_thresh, md = row
        mode, md = MODES[int(mode)], int(md)
        d = detector(C, mode, int(top_k), int(max_dets), float(nms), float(conf_thresh))
        check_call(d, loc, conf, mask[..., :md], priors, golden_wants(g, "case%d" % i, 3, md), mode)


@pytest.mark.parametrize("mode", MODES)
def test_golden_nan_inputs(g, mode):
    """A NaN foreground probability drops its prior (torch.max propagates NaN); a NaN box removes itself and every
    lower-scored box of its class in fast / cross-class NMS, and neither suppresses nor is suppressed in traditional."""
    loc, conf, mask, priors = (g["nan_" + k] for k in ("loc", "conf", "mask", "priors"))
    got = check_call(detector(21, mode), loc, conf, mask, priors, golden_wants(g, "nan_" + mode, 1, 8), mode)
    pr = prior_of(got[1][0, :int(got[4][0])])
    assert 5 not in pr and 6 not in pr


def test_nan_probability_at_class_two_or_more_drops_the_prior():
    """The probability form Detect.__call__ passes: a NaN at any foreground class >= 2 in a row whose max is above the
    threshold, at every position of the class loop."""
    r = np.random.RandomState(1)
    P, C = 300, 21
    loc, mask, priors = base_inputs(r, P)
    conf = np.full((1, P, C), 1e-3, np.float32)
    conf[0, :, 1] = r.uniform(0.06, 0.9, P).astype(np.float32)
    for j, c in enumerate(range(2, C)):
        conf[0, 10 * j, c] = np.nan
    for mode in MODES:
        d = detector(C, mode)
        got, _ = run(d, loc, conf, with_index_column(mask), priors)
        pr = prior_of(got[1][0, :int(got[4][0])])
        assert not np.isin(pr, 10 * np.arange(C - 2)).any(), mode
        check_image(got, 0, oracle(loc[0], conf[0], with_index_column(mask)[0], priors, mode), loc[0])


def test_nan_logit_drops_the_row():
    r = np.random.RandomState(2)
    P, C = 200, 21
    loc, mask, priors = base_inputs(r, P)
    logits = r.standard_normal((1, P, C)).astype(np.float32)
    logits[0, :, 3] += 5
    for j in range(0, P, 7):
        logits[0, j, j % C] = np.nan
    for mode in MODES:
        got, _ = run(detector(C, mode), loc, logits, with_index_column(mask), priors, logits=True)
        pr = prior_of(got[1][0, :int(got[4][0])])
        assert got[4][0] > 0 and not np.isin(pr, np.arange(0, P, 7)).any(), mode


def test_refusals():
    r = np.random.RandomState(3)
    loc, mask, priors = base_inputs(r, 64)
    conf = np.full((1, 64, 130), 0.1, np.float32)
    with pytest.raises(_lib.YbError):
        run(detector(130, "fast"), loc, conf, mask, priors)
    conf = conf[..., :81]
    with pytest.raises(_lib.YbError):
        run(detector(81, "fast", top_k=257), loc, conf, mask, priors)
    for mode in ("fast", "trad"):
        with pytest.raises(_lib.YbError):
            run(detector(81, mode), loc, conf, mask, priors, max_out=99)
    for mode in ("cc", "trad"):
        with pytest.raises(_lib.YbError):
            run(detector(81, mode), loc, conf, mask, priors, flags=_lib.YB_NMS_FLAG_SECOND_THRESHOLD)
    with pytest.raises(_lib.YbError):
        run(detector(81, "trad", top_k=50, max_dets=100), loc, conf, mask, priors)
    run(detector(81, "fast"), loc, conf, mask, priors)    # the launcher still works after its refusals


# ---------------------------------------------------------------------------------------------------------------------
# selection
# ---------------------------------------------------------------------------------------------------------------------
def base_inputs(r, P, B=1):
    """Priors on a 256 x 256 grid of disjoint 1/512 boxes (loc = 0 decodes them exactly) and random coefficients."""
    g = np.arange(P)
    priors = np.stack([(g % 256 + 0.5) / 256, (g // 256 % 256 + 0.5) / 256, np.full(P, 1 / 512), np.full(P, 1 / 512)],
                      1).astype(np.float32)
    return np.zeros((B, P, 4), np.float32), r.standard_normal((B, P, 4)).astype(np.float32), priors


def scores_conf(s, C=3, low=None):
    """Probabilities with class 1 = s (the scores under test); the other classes hold small distinct values."""
    P = s.shape[0]
    conf = np.zeros((1, P, C), np.float32)
    conf[0, :, 0] = 0.01
    conf[0, :, 1] = s
    for c in range(2, C):
        conf[0, :, c] = (np.arange(P) + 1 + c * P).astype(np.float32) * np.float32(2.0 ** -30) if low is None else low
    return conf


def keys(s, cand):
    """K2's 64-bit keys (score bits, ~prior) of the candidates, descending."""
    p = np.nonzero(cand)[0].astype(np.uint64)
    k = (s[cand].view(np.uint32).astype(np.uint64) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - p)
    return np.sort(k)[::-1]


PASS_FIELDS = [(53, 64), (42, 53), (32, 42), (21, 32), (10, 21), (0, 10)]


def deciding_pass(ks, K):
    """The radix pass whose digit separates the K-th key from the (K+1)-th."""
    h = int(ks[K - 1] ^ ks[K]).bit_length() - 1
    return [i for i, (lo, hi) in enumerate(PASS_FIELDS) if lo <= h < hi][0]


def cut_fixture(pass_, K, n, r):
    """Scores (class 1) for n candidates whose K-th and (K+1)-th keys first differ in the digit of radix pass `pass_`,
    with every key in one bin at the passes before it."""
    if pass_ in (0, 1, 2):
        if pass_ == 0:
            bits = np.concatenate([0x3F000000 + r.choice(1 << 21, K, replace=False),        # [0.5, 0.625)
                                   0x3E800000 + r.choice(1 << 21, n - K, replace=False)])   # [0.25, 0.3125)
        elif pass_ == 1:
            f = np.concatenate([r.choice(np.arange(1024, 2048), K, replace=False), r.choice(1024, n - K, replace=False)])
            bits = 0x3F000000 + (f << 10) + r.randint(0, 1024, n)
        else:
            f = np.concatenate([r.choice(np.arange(512, 1024), K, replace=False), r.choice(512, n - K, replace=False)])
            bits = 0x3F000000 + (77 << 10) + f
        s = bits.astype(np.uint32).view(np.float32)
        P = n
        full = s[r.permutation(n)]
    else:
        # equal scores: the prior index decides; pass 4 splits the K-th / (K+1)-th prior at a 1024 boundary
        start = 1024 - K if pass_ == 4 else 1030
        P = start + n + 50
        full = np.zeros(P, np.float32)
        full[start:start + n] = np.float32(0.625)
    return full, P


@pytest.mark.parametrize("pass_", [0, 1, 2, 4, 5])
@pytest.mark.parametrize("top_k", [200, 256])
def test_radix_cut_in_each_pass(pass_, top_k):
    r = np.random.RandomState(10 * pass_ + top_k)
    s, P = cut_fixture(pass_, top_k, 2 * top_k + 37, r)
    conf = scores_conf(s)
    cand = conf[0, :, 1:].max(1) > np.float32(0.05)
    assert deciding_pass(keys(s, cand), top_k) == pass_
    loc, mask, priors = base_inputs(r, P)
    for mode in ("fast", "cc"):
        d = detector(3, mode, top_k=top_k, max_dets=100)
        m = with_index_column(mask)
        got, _ = run(d, loc, conf, m, priors)
        check_image(got, 0, oracle(loc[0], conf[0], m[0], priors, mode, top_k=top_k), loc[0])


@pytest.mark.parametrize("top_k", [1, 200, 256])
@pytest.mark.parametrize("dm", [-1, 0, 1])
def test_candidate_count_around_top_k(top_k, dm):
    r = np.random.RandomState(top_k + dm)
    M = top_k + dm          # 0 for top_k = 1, dm = -1: no candidate at all
    P = M + 40
    s = np.zeros(P, np.float32)
    s[r.choice(P, M, replace=False)] = r.uniform(0.06, 0.99, M).astype(np.float32)
    loc, mask, priors = base_inputs(r, P)
    conf = scores_conf(s)
    assert (conf[0, :, 1:].max(1) > np.float32(0.05)).sum() == M
    for mode in MODES:
        md = min(100, top_k)
        d = detector(3, mode, top_k=top_k, max_dets=md)
        m = with_index_column(mask)
        got, _ = run(d, loc, conf, m, priors)
        check_image(got, 0, oracle(loc[0], conf[0], m[0], priors, mode, top_k=top_k, max_dets=md), loc[0])


def test_all_scores_equal_at_full_size():
    """P = 57744 equal scores: the lowest prior indices win, which only radix passes 4 and 5 can decide."""
    r = np.random.RandomState(4)
    P = 57744
    s = np.full(P, np.float32(0.6), np.float32)
    loc, mask, priors = base_inputs(r, P)
    conf = scores_conf(s, low=np.float32(0.001))
    for mode in MODES:
        d = detector(3, mode)
        m = with_index_column(mask)
        got, _ = run(d, loc, conf, m, priors)
        want = oracle(loc[0], conf[0], m[0], priors, mode)
        check_image(got, 0, want, loc[0])
        if mode != "cc":
            assert np.array_equal(prior_of(got[1][0, :100])[got[2][0, :100] == 0], np.arange(100))


@pytest.mark.parametrize("kind", ["tie_group_across_cut", "one_ulp_apart"])
def test_ties_and_ulps_at_the_cut(kind):
    r = np.random.RandomState(5)
    P, K = 700, 200
    s = r.uniform(0.1, 0.9, P).astype(np.float32)
    order = np.argsort(-s, kind="stable")
    if kind == "tie_group_across_cut":
        s[order[K - 5:K + 6]] = s[order[K - 5]]            # 11 equal scores, ranks K-5 .. K+5
    else:
        base = s[order[K - 20]]
        s[order[K - 20:K + 20]] = (base.view(np.uint32) - np.arange(40, dtype=np.uint32)).view(np.float32)
    loc, mask, priors = base_inputs(r, P)
    conf = scores_conf(s)
    for mode in MODES:
        d = detector(3, mode, top_k=K, max_dets=100)
        m = with_index_column(mask)
        got, _ = run(d, loc, conf, m, priors)
        check_image(got, 0, oracle(loc[0], conf[0], m[0], priors, mode, top_k=K), loc[0])


@pytest.mark.parametrize("P", [1, 127, 128, 129])
def test_priors_around_the_k1_tile(P):
    r = np.random.RandomState(P)
    priors = np.concatenate([r.uniform(0.2, 0.8, (P, 2)), r.uniform(0.05, 0.4, (P, 2))], 1).astype(np.float32)
    loc = (r.standard_normal((2, P, 4)) * 0.4).astype(np.float32)
    loc[:, ::2, 2:] = 0
    logits = (r.standard_normal((2, P, 21)) * 2).astype(np.float32)
    conf = O.softmax_rows(logits)
    conf[1, :, 0] = 1.0          # no candidates in image 1
    conf[1, :, 1:] = 0.01
    mask = r.standard_normal((2, P, 8)).astype(np.float32)
    for mode in MODES:
        m = with_index_column(mask)
        wants = [oracle(loc[b], conf[b], m[b], priors, mode, top_k=200) for b in range(2)]
        check_call(detector(21, mode), loc, conf, mask, priors, [None if w is None else dict(w, mask=w["mask"][:, :8])
                                                                  for w in wants], mode)


def trad_fixture(n, pairs, equal_from=None):
    """n class-1 candidates on disjoint boxes, scores descending with the prior index; each (i, j) in `pairs` moves
    rank j's box onto rank i's.  equal_from: ranks from there on share one score."""
    s = np.linspace(0.95, 0.2, n).astype(np.float32)
    if equal_from is not None:
        s[equal_from:] = s[equal_from]
    r = np.random.RandomState(n)
    loc, mask, priors = base_inputs(r, n)
    for i, j in pairs:
        priors[j] = priors[i]
        priors[j, 0] += np.float32(1 / 4096)
    return loc, scores_conf(s), mask, priors


@pytest.mark.parametrize("n", [256, 257, 300])
def test_trad_walk_across_the_chunk_boundary(n):
    """A suppressor in the first 256-key chunk and its victim in the second (rank 256 when n = 257); three suppressed
    boxes in the first chunk keep the walk going."""
    loc, conf, mask, priors = trad_fixture(n, [(3, 4), (10, 11), (20, 21), (7, n - 1)])
    d = detector(3, "trad", top_k=256, max_dets=256)
    m = with_index_column(mask)
    got, _ = run(d, loc, conf, m, priors)
    want = oracle(loc[0], conf[0], m[0], priors, "trad", top_k=256, max_dets=256)
    check_image(got, 0, want, loc[0])
    assert n - 1 not in prior_of(got[1][0, :int(got[4][0])])


def test_trad_equal_scores_across_the_chunk_boundary():
    loc, conf, mask, priors = trad_fixture(300, [(2, 5), (250, 258), (254, 257)], equal_from=248)
    d = detector(3, "trad", top_k=256, max_dets=256)
    m = with_index_column(mask)
    got, _ = run(d, loc, conf, m, priors)
    check_image(got, 0, oracle(loc[0], conf[0], m[0], priors, "trad", top_k=256, max_dets=256), loc[0])


def test_trad_more_survivors_than_max_dets():
    loc, conf, mask, priors = trad_fixture(150, [])
    m = with_index_column(mask)
    got, _ = run(detector(3, "trad", top_k=200, max_dets=100), loc, conf, m, priors)
    check_image(got, 0, oracle(loc[0], conf[0], m[0], priors, "trad"), loc[0])
    assert np.array_equal(prior_of(got[1][0]), np.arange(100))


@pytest.mark.parametrize("C", [2, 96, 97, 129])
def test_class_counts_at_full_size(C):
    """The class counts whose K1 tile needs more than 48 KB of shared memory, at P = 19248 against the oracle."""
    r = np.random.RandomState(C)
    P = 19248
    logits = (r.standard_normal((1, P, C)) * 2).astype(np.float32)
    logits[:, :, 0] += 4.0
    priors = np.concatenate([r.uniform(0.05, 0.95, (P, 2)), r.uniform(0.02, 0.5, (P, 2))], 1).astype(np.float32)
    loc = r.standard_normal((1, P, 4)).astype(np.float32)
    loc[:, ::3, 2:] = 0
    mask = r.standard_normal((1, P, 4)).astype(np.float32)
    conf = O.softmax_rows(logits)
    for mode in MODES:
        m = with_index_column(mask)
        got, _ = run(detector(C, mode), loc, conf, m, priors)
        check_image(got, 0, oracle(loc[0], conf[0], m[0], priors, mode), loc[0])


# ---------------------------------------------------------------------------------------------------------------------
# thresholds
# ---------------------------------------------------------------------------------------------------------------------
def test_conf_threshold_probabilities():
    """Best foreground probability exactly float32(t): not a candidate (`>`); the next float up: a candidate."""
    for t in (0.05, 0.5):
        r = np.random.RandomState(6)
        P = 64
        s = np.full(P, np.float32(0.001))
        s[10], s[20] = np.float32(t), np.nextafter(np.float32(t), np.float32(1))
        loc, mask, priors = base_inputs(r, P)
        conf = scores_conf(s, C=2)
        for mode in MODES:
            got, _ = run(detector(2, mode, conf_thresh=t), loc, conf, with_index_column(mask), priors)
            assert list(prior_of(got[1][0, :int(got[4][0])])) == [20], (t, mode)


def test_conf_threshold_logits():
    """The fused-softmax form.  For C = 2 yb_softmax is K1's softmax bit for bit (one max, one sum of two terms), so it
    names the rows whose probability is exactly a threshold p* and the next float up; p* is the produced value nearest
    t whose upper neighbour is produced too."""
    lib = _lib.load()
    for t in (0.05, 0.5):
        P = 4096
        d0 = np.float32(np.log(t / (1 - t))) if t != 0.5 else np.float32(0)
        k = np.arange(P) - P // 2
        dl = (d0.view(np.int32) + k).astype(np.int32).view(np.float32) if t != 0.5 else \
            (k * 2.0 ** -26).astype(np.float32)
        logits = np.zeros((1, P, 2), np.float32)
        logits[0, :, 1] = dl
        x = torch.from_numpy(logits).cuda()
        p = torch.empty_like(x)
        d = detector(2, "cc", top_k=256, nms=1.0, conf_thresh=t)
        _lib.check(lib.yb_softmax(d._handle(x.device), _lib.ptr(x), _lib.ptr(p), P, 2, _lib.current_stream()), "softmax")
        p1 = p.cpu().numpy()[0, :, 1]
        vals = np.unique(p1)
        # p*: produced, nearest t, preferably with its upper float neighbour produced too
        up = vals[:-1][np.nextafter(vals[:-1], np.float32(1)) == vals[1:]]
        ps = (up if up.size else vals[:-1])[np.argmin(np.abs((up if up.size else vals[:-1]).astype(np.float64) - t))]
        nxt = vals[np.searchsorted(vals, ps) + 1]
        at, above = np.nonzero(p1 == ps)[0][:1], np.nonzero(p1 == nxt)[0][:1]
        sel = np.concatenate([at, above])
        r = np.random.RandomState(7)
        loc, mask, priors = base_inputs(r, 2)
        d = detector(2, "cc", top_k=256, nms=1.0, conf_thresh=float(ps))
        got, _ = run(d, loc, logits[:, sel], with_index_column(mask), priors, logits=True)
        assert int(got[4][0]) == 1 and prior_of(got[1][0, :1])[0] == 1 and got[3][0, 0] == nxt, t
        print("conf_thresh %.2f, logits: p* = %.9g, next produced %s" % (t, ps, "float up" if up.size else "value"))


def f32(x):
    return np.float32(x)


def fma(a, b, c):
    """fp32 fused multiply-add (one rounding; the exact product of two fp32 values fits a float64)."""
    return np.float32(np.float64(a) * np.float64(b) + np.float64(c))


def decode32(loc, pri, contract=False):
    """detect.cu's decode_box in fp32; contract=True: what nvcc makes of it with FMA contraction."""
    t0, t1 = f32(loc[0] * f32(0.1)), f32(loc[1] * f32(0.1))
    if contract:
        cx, cy = fma(t0, pri[2], pri[0]), fma(t1, pri[3], pri[1])
    else:
        cx, cy = f32(pri[0] + f32(t0 * pri[2])), f32(pri[1] + f32(t1 * pri[3]))
    w = f32(pri[2] * f32(np.exp(np.float64(f32(loc[2] * f32(0.2))))))
    h = f32(pri[3] * f32(np.exp(np.float64(f32(loc[3] * f32(0.2))))))
    x1, y1 = f32(cx - f32(w / f32(2))), f32(cy - f32(h / f32(2)))
    return np.array([x1, y1, f32(x1 + w), f32(y1 + h)], np.float32)


def iou32(a, b, contract=False):
    iw = max(f32(min(a[2], b[2]) - max(a[0], b[0])), f32(0))
    ih = max(f32(min(a[3], b[3]) - max(a[1], b[1])), f32(0))
    inter = f32(iw * ih)
    wa, ha, wb, hb = f32(a[2] - a[0]), f32(a[3] - a[1]), f32(b[2] - b[0]), f32(b[3] - b[1])
    if contract:      # area_a + area_b -> fma(wa, ha, area_b); (...) - inter -> fma(-iw, ih, ...)
        return f32(inter / fma(-iw, ih, fma(wa, ha, f32(wb * hb))))
    return f32(inter / f32(f32(f32(wa * ha) + f32(wb * hb)) - inter))


def iou64(a, b):
    a, b = a.astype(np.float64), b.astype(np.float64)
    iw = max(min(a[2], b[2]) - max(a[0], b[0]), 0)
    ih = max(min(a[3], b[3]) - max(a[1], b[1]), 0)
    inter = iw * ih
    return inter / ((a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - inter)


def dyadic_pair(t):
    """(priors of A, priors of B) whose fp32 IoU is exactly float32(t).  Coordinates are
    multiples of 2^-30 below 2^-8 with height 2^-9, so decode, areas and union are exact and the IoU is one correctly
    rounded division i / U of integers."""
    u, H = 2.0 ** -30, 2.0 ** -9
    U = next(U for U in range(1 << 21, 1 << 22) if round(t * U) == t * U and (U + round(t * U)) % 2 == 0)
    i = round(t * U)          # i / U == t exactly as rationals (t = 3/10, 1/2, 7/10): fl32(i / U) == float32(t)
    a = (U + i) // 2          # both widths
    ax1, bx1 = 2 * u * 64, 2 * u * 64 + (a - i) * u
    pa = [ax1 + a * u / 2, H, a * u, H]
    pb = [bx1 + a * u / 2, H, a * u, H]
    return np.array(pa, np.float32), np.array(pb, np.float32)


def swept_pairs(t, n, r):
    """n pairs whose IoU lands within a few ulp of t through an inexact decode (loc[0] != 0): same-size boxes, B shifted
    right by w (1 - t) / (1 + t) through its loc."""
    pairs = []
    for _ in range(n):
        w, h = r.uniform(0.1, 0.3), r.uniform(0.1, 0.3)
        cx, cy = r.uniform(0.3, 0.5), r.uniform(0.3, 0.7)
        pa = np.array([cx, cy, w, h], np.float32)
        pb = np.array([cx + r.uniform(-0.01, 0.01), cy, w, h], np.float32)
        shift = w * (1 - t) / (1 + t)
        lb = np.array([(cx + shift - pb[0]) / (0.1 * pb[2]), 0, 0, 0], np.float32)
        pairs.append((pa, pb, lb))
    return pairs


@pytest.mark.parametrize("t", [0.3, 0.5, 0.7])
def test_iou_threshold_fast_and_cc(t):
    """Two candidates per image, B higher scored: kept by fast / cc when IoU <= float32(t).  Dyadic pairs at exactly
    float32(t), plus swept pairs whose inexact decode lands within a few ulp either side."""
    r = np.random.RandomState(int(t * 10))
    images = [dyadic_pair(t) + (np.zeros(4, np.float32),)] + swept_pairs(t, 300, r)
    B = len(images)
    priors = np.concatenate([np.stack([pa, pb]) for pa, pb, _ in images]).astype(np.float32)
    P = priors.shape[0]
    loc = np.zeros((B, P, 4), np.float32)
    conf = np.zeros((B, P, 2), np.float32)
    conf[:, :, 0] = 1
    for b, (_, _, lb) in enumerate(images):
        loc[b, 2 * b + 1] = lb
        conf[b, 2 * b, :] = [0.1, 0.9]
        conf[b, 2 * b + 1, :] = [0.2, 0.8]
    mask = np.zeros((B, P, 3), np.float32)
    tv = f32(t)
    near = flips = 0
    for mode in ("fast", "cc"):
        got, _ = run(detector(2, mode, nms=t), loc, conf, with_index_column(mask), priors)
        for b in range(B):
            a, bb = decode32(loc[b, 2 * b], priors[2 * b]), decode32(loc[b, 2 * b + 1], priors[2 * b + 1])
            iou = iou32(a, bb)
            kept = int(got[4][b]) == 2
            assert kept == (iou <= tv), (mode, b, iou, tv)
            if b == 0:
                assert iou == tv and kept
            if mode == "fast":
                margin = (iou64(a, bb) - np.float64(tv)) / np.spacing(tv)
                near += abs(margin) <= 1
                ac, bc = decode32(loc[b, 2 * b], priors[2 * b], True), decode32(loc[b, 2 * b + 1], priors[2 * b + 1], True)
                flips += (iou32(ac, bc, True) <= tv) != kept
            check_image(got, b, oracle(loc[b], conf[b], with_index_column(mask)[b], priors, mode, nms=t), loc[b])
    # the float64 audit: decisions within one fp32 ulp of the threshold, and an FMA-contracted decode / IoU changes at
    # least one of them; otherwise these fixtures could no longer tell the kernel's arithmetic from a contracted one
    print("nms_thresh %.1f: %d of %d decisions within 1 ulp of the threshold, %d flipped by FMA contraction" %
          (t, near, B, flips))
    assert near >= 5 and flips >= 1


@pytest.mark.parametrize("t", [0.3, 0.5, 0.7])
def test_iou_threshold_traditional(t):
    """cython_nms's `ovr >= thresh` on boxes scaled by max_size with the +1 pixel convention: with max_size = 512 and
    pixel-integer boxes of equal height the overlap is exactly iw / (Wa + Wb - iw) correctly rounded, so a pair at
    t = 3/10, 1/2, 7/10 sits exactly on float32(t) and is suppressed."""
    iw, W = {0.3: (6, 13), 0.5: (2, 3), 0.7: (14, 17)}[t]
    ax1 = 100
    bx1 = ax1 + W - iw
    px = lambda x1: [(x1 + (W - 1) / 2) / 512, 200 / 512, (W - 1) / 512, 30 / 512]
    pairs = [(px(ax1), px(bx1)), (px(ax1), px(bx1 + 1))]
    B = len(pairs)
    priors = np.array([p for pr in pairs for p in pr], np.float32)
    P = priors.shape[0]
    loc = np.zeros((B, P, 4), np.float32)
    conf = np.zeros((B, P, 2), np.float32)
    conf[:, :, 0] = 1
    for b in range(B):
        conf[b, 2 * b, :] = [0.1, 0.9]
        conf[b, 2 * b + 1, :] = [0.2, 0.8]
    mask = np.zeros((B, P, 3), np.float32)
    got, _ = run(detector(2, "trad", nms=t, max_size=512), loc, conf, with_index_column(mask), priors)
    assert int(got[4][0]) == 1 and int(got[4][1]) == 2, t          # exactly at the threshold: suppressed
    for b in range(B):
        check_image(got, b, oracle(loc[b], conf[b], with_index_column(mask)[b], priors, "trad", nms=t, max_size=512),
                    loc[b])


# ---------------------------------------------------------------------------------------------------------------------
# fused softmax
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [2, 21, 81, 129])
def test_fused_softmax_scores(C):
    """Every output score above conf_thresh of the logits path against a float64 softmax, within (C + 2) u relative,
    u = 2^-24.  K1 computes e_c = expf(x_c - m), s = a sequential fp32 sum of the C positive e_c and e_c / s.  To first
    order: the sum of positive terms adds at most (C - 1) u relative (one rounding per partial sum, each bounded by the
    final s); the division one u; expf, 2 ulp, counted as 2 u on e_c (the max term is exactly expf(0) = 1, and the
    terms that dominate s and the reported e_c are within a factor ln 20 of it for scores above 0.05)."""
    r = np.random.RandomState(C + 1)
    P = 3000
    logits = (r.standard_normal((1, P, C)) * 3).astype(np.float32)
    logits[:, :, 0] += 2
    loc = np.zeros((1, P, 4), np.float32)
    priors = np.concatenate([r.uniform(0.1, 0.9, (P, 2)), r.uniform(0.05, 0.3, (P, 2))], 1).astype(np.float32)
    mask = np.zeros((1, P, 3), np.float32)
    x = logits[0].astype(np.float64)
    e = np.exp(x - x.max(1, keepdims=True))
    p64 = e / e.sum(1, keepdims=True)
    for mode in ("fast", "cc"):
        got, _ = run(detector(C, mode), loc, logits, with_index_column(mask), priors, logits=True)
        n = int(got[4][0])
        assert n > 0
        pr = prior_of(got[1][0, :n])
        want = p64[pr, got[2][0, :n] + 1] if mode == "fast" else p64[pr, 1:].max(1)
        above = got[3][0, :n] > np.float32(0.05)
        assert above.sum() > 0
        ratio = np.abs(got[3][0, :n] - want)[above] / (want[above] * (C + 2) * U24)
        SOFTMAX_RATIO.append(float(ratio.max()))
        assert ratio.max() <= 1, (mode, float(ratio.max()))
