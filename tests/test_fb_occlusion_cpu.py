"""The forward-backward occlusion check's restatement (tests/fb_ref.py) on analytic cases, the refusals of run --backward and
evaluate --fb-check before any device work, the derived-path collisions, the 8-bit grey PNG writer, and the KITTI and RGB
writers' bytes."""
import hashlib
import re
import zlib

import numpy as np
import pytest

from flownet2_b200 import evaluate as E
from flownet2_b200 import kitti as K
from flownet2_b200 import run as R
from tests import fb_ref as ref
from tests.test_run_flownet_cpu import write_pnm


def uniform(H, W, u, v):
    f = np.empty((H, W, 2), np.float32)
    f[..., 0], f[..., 1] = u, v
    return f


def test_zero_flows_mark_nothing():
    z = np.zeros((7, 9, 2), np.float32)
    assert (ref.fb_occlusion(z, z) == 0).all()
    assert (ref.fb_occlusion(z, z, 0.0, 0.0) == 0).all()


@pytest.mark.parametrize("t", [(3, 0), (-2, 0), (0, 4), (5, -3), (2.5, 1.25)])
def test_translation_marks_what_leaves(t):
    H, W = 11, 16
    tx, ty = t
    got = ref.fb_occlusion(uniform(H, W, tx, ty), uniform(H, W, -tx, -ty))
    ys, xs = np.mgrid[0:H, 0:W]
    x2, y2 = xs + tx, ys + ty
    want = (x2 < 0) | (x2 >= W) | (y2 < 0) | (y2 >= H)
    assert np.array_equal(got == 255, want) and want.any() and (~want).any()
    assert set(np.unique(got)) <= {0, 255}


@pytest.mark.parametrize("d", [1, 3, 6])
def test_moving_square_marks_the_covered_strip(d):
    H, W, y0, x0, s = 20, 30, 5, 6, 8
    fwd = np.zeros((H, W, 2), np.float32)
    fwd[y0:y0 + s, x0:x0 + s, 0] = d                                   # the square moves d px right
    bwd = np.zeros((H, W, 2), np.float32)
    bwd[y0:y0 + s, x0 + d:x0 + d + s, 0] = -d                           # where it is in frame 1, back
    got = ref.fb_occlusion(fwd, bwd)
    want = np.zeros((H, W), bool)
    want[y0:y0 + s, x0 + s:x0 + s + d] = True                           # the background the square covers in frame 1
    assert np.array_equal(got == 255, want)


def test_non_finite_is_occluded():
    H, W = 6, 7
    fwd, bwd = np.zeros((H, W, 2), np.float32), np.zeros((H, W, 2), np.float32)
    fwd[1, 2] = (np.nan, 0)
    fwd[2, 3] = (0, np.inf)
    fwd[3, 1] = (-np.inf, 0)
    # A non-finite backward value makes every sample that has it among its four taps non-finite, at weight 0 too (FlowWarp's
    # mix multiplies it): with zero flow, pixel (y, x) has the taps (y, x), (y, x + 1), (y + 1, x), (y + 1, x + 1).
    bwd[4, 5] = (np.nan, 0)
    fwd[0, 0] = (1.5, 0)                                               # lands between (0, 1) and (0, 2)
    bwd[0, 2] = (0, np.inf)                                            # its tap of weight 0.5
    got = ref.fb_occlusion(fwd, bwd)
    want = np.zeros((H, W), bool)
    for y, x in ((1, 2), (2, 3), (3, 1), (4, 5), (4, 4), (3, 5), (3, 4), (0, 2), (0, 1), (0, 0)):
        want[y, x] = True
    assert np.array_equal(got == 255, want)


def test_alpha2_sets_the_threshold_for_tiny_flows():
    H, W = 5, 6
    z = np.zeros((H, W, 2), np.float32)
    b = uniform(H, W, 0.6, 0.0)                                        # lhs = mag = 0.36 in float32
    lhs = np.float32(0.6) * np.float32(0.6)
    assert (ref.fb_occlusion(z, b, 0.0, float(lhs)) == 0).all()       # not above
    assert (ref.fb_occlusion(z, b, 0.0, float(np.nextafter(lhs, np.float32(0)))) == 255).all()
    assert (ref.fb_occlusion(z, b, 0.01, 0.5) == 0).all()
    assert (ref.fb_occlusion(z, b, 0.01, 0.35) == 255).all()


def test_warp_restatement_matches_flowwarp_taps():
    """Sampling a linear ramp bilinearly is exact enough to recover the landing point."""
    H, W = 9, 12
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float32)
    img = np.stack([xs, ys], -1)
    f = uniform(H, W, 0.25, 0.5)
    out, inside = ref.warp(img, f)
    assert np.array_equal(inside, (xs + 0.25 < W) & (ys + 0.5 < H))
    interior = (xs + 1 < W) & (ys + 1 < H)                              # all four taps inside: no clamping
    assert np.allclose(out[interior], np.stack([xs + 0.25, ys + 0.5], -1)[interior], atol=1e-6)
    assert (out[~inside] == 0).all()


# ---- refusals, before any device work ----
@pytest.fixture
def no_device(monkeypatch):
    """Fails a test that reaches the device."""
    def boom(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(R, "run_groups", boom)
    monkeypatch.setattr(E, "run_groups", boom)
    import torch
    monkeypatch.setattr(torch.cuda, "set_device", boom)


@pytest.mark.parametrize("flag", ["--fb-alpha1", "--fb-alpha2"])
@pytest.mark.parametrize("value", ["-0.1", "nan", "inf", "-inf"])
def test_alphas_refused(tmp_path, capsys, no_device, flag, value):
    assert R.main(["w", "t", "a", "b", "o.flo", "--backward", flag + "=" + value]) == 2
    assert E.main(["w", "t", "l", "--fb-check", flag + "=" + value]) == 2
    err = capsys.readouterr().err.strip().splitlines()
    assert len(err) == 2 and all(flag + " must be a finite non-negative number" in e for e in err)
    kw = {"fb_alpha1": float(value)} if flag == "--fb-alpha1" else {"fb_alpha2": float(value)}
    with pytest.raises(R.RunError, match="must be a finite non-negative number"):
        R.run("w", "t", [], backward=True, **kw)
    fb = (float(value), 0.5) if flag == "--fb-alpha1" else (0.01, float(value))
    with pytest.raises(R.RunError, match="must be a finite non-negative number"):
        E.evaluate(str(tmp_path / "none.caffemodel"), "t", [], fb=fb)


def test_alpha_zero_accepted():
    R.check_fb_alphas(0.0, 0.0)
    R.check_fb_alphas(0.01, 0.5)


def test_derived_paths():
    assert R.bwd_path("a/b.flo") == "a/b.bwd.flo" and R.bwd_path("x.png") == "x.bwd.png" and R.bwd_path("noext") == "noext.bwd"
    assert R.occ_path("a/b.flo") == "a/b.occ.png" and R.occ_path("x.png") == "x.occ.png"
    assert R.derived_paths(False, False) == ()
    assert R.derived_paths(True, True) == (R.vis_path, R.bwd_path, R.occ_path)


def test_colliding_derived_paths_refused(tmp_path, capsys, no_device):
    a = write_pnm(tmp_path / "a.ppm", np.zeros((8, 8, 3), np.uint8))
    b = write_pnm(tmp_path / "b.ppm", np.zeros((8, 8, 3), np.uint8))
    w, t = tmp_path / "w.caffemodel", tmp_path / "t.template"
    w.write_bytes(b"")
    t.write_text("")
    lst = tmp_path / "l.txt"
    cases = [(("x.flo", "x.png"), [], "both have the occlusion mask"),
             (("y.flo", "y.bwd.flo"), [], "the backward flow .* is the output of"),
             (("z.flo", "z.occ.png"), [], "the occlusion mask .* is the output of"),
             (("v.flo", "v.vis.png"), ["--visualize"], "the visualisation .* is the output of"),
             (("p.flo", "p.png"), ["--visualize"], "both visualise to")]
    for outs, extra, what in cases:
        lst.write_text("".join("%s %s %s\n" % (a, b, tmp_path / o) for o in outs))
        pairs = R.read_list(str(lst), ground_truth=False)
        assert R.main([str(w), str(t), str(lst), "--backward"] + extra) == 2
        err = capsys.readouterr().err
        assert re.search(what, err) and err.count("\n") == 1, (outs, err)
        with pytest.raises(R.RunError, match=what):
            R.run(str(w), str(t), pairs, backward=True, visualize=bool(extra))
    # without --backward the same lists pass the visualisation check as before
    lst.write_text("%s %s %s\n%s %s %s\n" % (a, b, tmp_path / "y.flo", a, b, tmp_path / "y.bwd.flo"))
    R.check_vis_paths(R.read_list(str(lst), ground_truth=False))
    # one output listed twice: one set of files
    lst.write_text("%s %s %s\n%s %s %s\n" % (a, b, tmp_path / "z.flo", a, b, tmp_path / "z.flo"))
    R.check_vis_paths(R.read_list(str(lst), ground_truth=False), R.derived_paths(True, True))


# ---- PNG writers ----
def test_grey_png_round_trip(tmp_path):
    r = np.random.default_rng(3)
    H, W = 13, 21
    mask = np.where(r.random((H, W)) < 0.3, 255, 0).astype(np.uint8)
    rows = np.concatenate([np.zeros((H, 1), np.uint8), mask], 1)       # filter None
    path = K.write_png_rows(str(tmp_path / "m.png"), rows, W, H, 8, 1)
    data = open(path, "rb").read()
    assert data[:8] == K.SIGNATURE and (data[24], data[25]) == (8, 0)  # bit depth 8, grey
    assert zlib.decompress(K._idat(path, data)) == rows.tobytes()
    try:
        from PIL import Image
    except ImportError:
        return
    with Image.open(path) as im:
        assert im.mode == "L" and np.array_equal(np.asarray(im), mask)


def test_rgb_and_kitti_png_bytes_unchanged():
    """The RGB and KITTI writers' bytes for these rows were hashed before the writer took a channel count."""
    r = np.random.default_rng(5)
    r.integers(0, 256, (11, 51), dtype=np.uint8)
    rows = np.concatenate([np.full((11, 1), 4, np.uint8), r.integers(0, 256, (11, 51), dtype=np.uint8)], 1)
    rows16 = np.concatenate([np.full((5, 1), 1, np.uint8), r.integers(0, 256, (5, 54), dtype=np.uint8)], 1)
    assert hashlib.sha256(K.png_bytes(rows.tobytes(), 17, 11, 8)).hexdigest() == \
        "80945fb11dfb1baf7ceeda2d752eb50fabb75651385df80f4ce828689944e281"
    assert hashlib.sha256(K.png_bytes(rows16.tobytes(), 9, 5)).hexdigest() == \
        "336193a4e77c2528df535c40ff7196f66e96b10b70f0a5bebe5c9ad30edec05d"
    assert K.png_bytes(rows.tobytes(), 17, 11, 8) == K.png_bytes(rows.tobytes(), 17, 11, 8, 3)
