"""2-D augmentation (Segmenation_Aug, dataprocess/AugData.py) without a GPU: the cv2 oracle (oracle/augment2d.py)
against fixtures recorded from cv2, the drop-in's host draws against the restated albumentations 1.1.0 sequence, the
motion kernels, the refusals, ``install()``, and the Python layer (``transform_compose``, ``DataAugmentation``,
``transform_batch``, ``InputStager(augment=...)``) on an emulated backend that runs csrc/augment2d.cu's rule in numpy
from the packed parameter table."""
import json
import os
import random
import struct
import sys
import types

import cv2
import numpy as np
import pytest
import torch

from oracle import augment2d as oa
from oracle import resize2d as RZ
from oracle import staging as OS
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import augment2d as A2
from pytorchdeeplearing_b200 import runtime
from pytorchdeeplearing_b200._abi import AUG2D_PARAM_BYTES
from conftest import GOLDEN
from emu_backend import EmuBackend

GOLD = np.load(os.path.join(GOLDEN, "augment2d.npz"))
META = json.loads(str(GOLD["meta"]))


def fixture_source(case):
    """a case's source: stored once per image, or the deterministic pattern for the large ones"""
    if case["src"] is not None:
        return GOLD[case["src"]]
    return oa.pattern_image(case["shape"][0], case["shape"][1], case["shape"][2] if len(case["shape"]) == 3 else 1)


def matches_fixture(i, out):
    """out equals case i's recorded bytes (the SHA-256 of them for the large cases)"""
    case = META[i]
    if "sha256" in case:
        return tuple(out.shape) == tuple(case["shape"]) and oa.digest(out) == case["sha256"]
    return np.array_equal(out, GOLD[f"out_{i}"])


def oracle_stage(case, src):
    st = case["stage"]
    if st == "flip":
        return oa.flip(src, case["hflip"], case["vflip"])
    if st == "motion":
        return oa.blur(src, "motion", np.array(case["kernel"], dtype=np.float32))
    if st in ("median", "box"):
        return oa.blur(src, st)
    if st in ("warp", "warp_mask"):
        return oa.warp(src, oa.ssr_matrix(src.shape[0], src.shape[1], *case["ssr"]), nearest=st == "warp_mask")
    return cv2.LUT(src, oa.bc_table(case["alpha"], case["beta"]))


@pytest.mark.parametrize("stage", ["flip", "motion", "median", "box", "warp", "warp_mask", "lut"])
def test_oracle_equals_the_cv2_fixtures(stage):
    n = 0
    for i, case in enumerate(META):
        if case["stage"] == stage:
            assert matches_fixture(i, oracle_stage(case, fixture_source(case))), (i, case)
            n += 1
    assert n >= 8


def test_fixtures_cover_the_issue_list():
    shapes = {tuple(c["shape"]) for c in META}
    assert {(512, 512), (512, 512, 3), (700, 1000), (1000, 700), (9, 1), (1, 1), (37, 53, 3)} <= shapes
    ks = {(c["k"], tuple(c["line"])) for c in META if c["stage"] == "motion"}
    for k in (3, 5, 7):
        lines = [ln for kk, ln in ks if kk == k]
        assert any(ys == ye for _, ys, _, ye in lines) and any(xs == xe for xs, _, xe, _ in lines)
        assert any(abs(xe - xs) == abs(ye - ys) for xs, ys, xe, ye in lines)
        assert any(abs(ye - ys) > abs(xe - xs) > 0 for xs, ys, xe, ye in lines)
    bcs = {(c["alpha"], c["beta"]) for c in META if c["stage"] == "lut"}
    assert {(0.7, 0.0), (1.3, 0.0), (1.0, 0.3), (1.0, -0.3), (1.0, 0.0)} <= bcs
    ssrs = [c["ssr"] for c in META if c["stage"] == "warp"]
    assert [45, 0.8, 0.0625, 0.0625] in ssrs and [-45, 1.2, -0.0625, -0.0625] in ssrs
    assert max(abs(s[2]) + abs(s[3]) for s in ssrs) > 2


@pytest.mark.parametrize("seed", range(40))
def test_drop_in_draws_consume_random_as_the_restatement(seed):
    random.seed(seed)
    want = [oa.draw() for _ in range(25)]
    state = random.getstate()
    random.seed(seed)
    got = [A2.draw_params() for _ in range(25)]
    assert random.getstate() == state
    for a, b in zip(want, got):
        for key in ("hflip", "vflip", "blur", "ssr", "bc"):
            assert a[key] == b[key]
        assert (a["kernel"] is None) == (b["kernel"] is None)
        if a["kernel"] is not None:
            assert a["kernel"].dtype == b["kernel"].dtype == np.float32 and np.array_equal(a["kernel"], b["kernel"])


def test_draw_sequence_reaches_every_stage():
    random.seed(3)
    draws = [A2.draw_params() for _ in range(3000)]
    assert {d["blur"] for d in draws} == {None, "motion", "median", "box"}
    assert {d["kernel"].shape[0] for d in draws if d["kernel"] is not None} == {3, 5, 7}
    frac = np.mean([d["ssr"] is not None for d in draws])
    assert 0.17 < frac < 0.23
    for d in draws:
        if d["ssr"] is not None:
            a, s, dx, dy = d["ssr"]
            assert -45 <= a <= 45 and 0.8 <= s <= 1.2 and abs(dx) <= 0.0625 and abs(dy) <= 0.0625


def test_motion_kernel_construction():
    k = oa.motion_kernel(5, 0, 2, 4, 2)
    assert k.dtype == np.float32 and np.array_equal(k[2], np.full(5, np.float32(0.2))) and k.sum(0).min() > 0
    k = oa.motion_kernel(7, 3, 0, 3, 6)
    assert np.count_nonzero(k) == 7 and np.count_nonzero(k[:, 3]) == 7
    k = oa.motion_kernel(3, 0, 0, 2, 2)
    assert np.array_equal(k, np.eye(3, dtype=np.float32) / np.float32(3))
    k = oa.motion_kernel(7, 0, 0, 2, 6)                                    # steep: one tap per row
    assert np.count_nonzero(k) == 7 and all(np.count_nonzero(r) == 1 for r in k)
    taps = A2.kernel_taps(oa.motion_kernel(5, 4, 0, 0, 4))
    assert [(dy, dx) for dy, dx, _ in taps] == [(-2, 2), (-1, 1), (0, 0), (1, -1), (2, -2)]
    assert all(w == np.float32(0.2) for _, _, w in taps)


def test_refusals():
    aug = b200.Segmenation_Aug()
    with pytest.raises(TypeError):
        aug.transform_compose(image=np.zeros((4, 4), np.float32))
    for shape in ((4, 4, 2), (4, 4, 4), (4,), (2, 4, 4, 3)):
        with pytest.raises(ValueError):
            aug.transform_compose(image=np.zeros(shape, np.uint8))
    with pytest.raises(ValueError):
        aug.transform_compose(image=np.zeros((4, 5, 3), np.uint8), mask=np.zeros((5, 4), np.uint8))
    with pytest.raises(TypeError):
        aug.transform_batch(torch.zeros(2, 4, 4))
    with pytest.raises(ValueError):
        aug.transform_batch(torch.zeros(2, 4, 4, 2, dtype=torch.uint8))
    with pytest.raises(ValueError):
        aug.transform_batch(torch.zeros(2, 4, 4, dtype=torch.uint8), torch.zeros(2, 4, 5, dtype=torch.uint8))
    with pytest.raises(ValueError):
        b200.InputStager("cpu", (2, 8, 8), backend=EmuAug(), augment=aug)


def test_install_rebinds_segmenation_aug_in_dataprocess_augdata():
    pkg = types.ModuleType("dataprocess")
    mod = types.ModuleType("dataprocess.AugData")

    class Orig:
        pass

    mod.Segmenation_Aug = Orig
    saved = {k: sys.modules.get(k) for k in ("dataprocess", "dataprocess.AugData")}
    sys.modules["dataprocess"], sys.modules["dataprocess.AugData"] = pkg, mod
    try:
        assert b200.install() == 1
        assert mod.Segmenation_Aug is b200.Segmenation_Aug
        b200.uninstall()
        assert mod.Segmenation_Aug is Orig
    finally:
        b200.uninstall()
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


# ---------------------------------------------------------------------------------------------- emulated backend
def refl(i, n):
    if n == 1:
        return np.zeros_like(i)
    i = np.asarray(i)
    while ((i < 0) | (i >= n)).any():
        i = np.where(i < 0, -i, i)
        i = np.where(i >= n, 2 * n - 2 - i, i)
    return i


def unpack(raw):
    f = struct.unpack("<4q6d8f8b8b8i", raw[:160])
    return dict(src=f[0], dst=f[1], msrc=f[2], mdst=f[3], minv=f[4:10], tap_w=f[10:18], tap_dy=f[18:26],
                tap_dx=f[26:34], h=f[34], w=f[35], c=f[36], flags=f[37], blur=f[38], ntaps=f[39], fcn=f[40],
                lut=np.frombuffer(raw[160:416], np.uint8))


def emu_blur(img, e):
    """flipped image (h, w, c) -> the blur of csrc/augment2d.cu, restated"""
    h, w, c = img.shape
    ys, xs = np.mgrid[0:h, 0:w]
    if e["blur"] == 1:
        s = np.zeros(img.shape, np.float32)
        s2 = np.zeros(img.shape, np.float32)
        for t in range(e["ntaps"]):
            v = img[refl(ys + e["tap_dy"][t], h), refl(xs + e["tap_dx"][t], w)].astype(np.float32)
            wt = np.float32(e["tap_w"][t])
            s = (v.astype(np.float64) * wt + s).astype(np.float32)          # fma: one rounding
            s2 = (s2 + v * wt).astype(np.float32)
        idx = xs[..., None] * e["fcn"] + np.arange(c)
        s = np.where(idx < ((w * e["fcn"]) & ~3), s, s2)
        return np.clip(np.rint(s), 0, 255).astype(np.uint8)
    if e["blur"] == 2:
        taps = [img[np.clip(ys + dy, 0, h - 1), np.clip(xs + dx, 0, w - 1)] for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
        return np.median(np.stack(taps), axis=0).astype(np.uint8)
    s = sum(img[refl(ys + dy, h), refl(xs + dx, w)].astype(np.int64) for dy in (-1, 0, 1) for dx in (-1, 0, 1))
    return ((2 * s + 9) // 18).astype(np.uint8)


def emu_warp(img, m, nearest):
    h, w = img.shape[:2]
    ys, xs = np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64)
    ax = np.rint(m[0] * xs * 1024).astype(np.int64)
    ay = np.rint(m[3] * xs * 1024).astype(np.int64)
    rx = np.rint((m[1] * ys + m[2]) * 1024).astype(np.int64)
    ry = np.rint((m[4] * ys + m[5]) * 1024).astype(np.int64)
    if nearest:
        return img[refl((ry[:, None] + 512 + ay[None]) >> 10, h), refl((rx[:, None] + 512 + ax[None]) >> 10, w)]
    X = (rx[:, None] + 16 + ax[None]) >> 5
    Y = (ry[:, None] + 16 + ay[None]) >> 5
    sx, sy, fx, fy = X >> 5, Y >> 5, (X & 31)[..., None], (Y & 31)[..., None]
    x0, x1, y0, y1 = refl(sx, w), refl(sx + 1, w), refl(sy, h), refl(sy + 1, h)
    p = img.astype(np.int64)
    s = (p[y0, x0] * (32 - fy) * (32 - fx) + p[y0, x1] * (32 - fy) * fx + p[y1, x0] * fy * (32 - fx) +
         p[y1, x1] * fy * fx) * 32
    return np.minimum((s + (1 << 14)) >> 15, 255).astype(np.uint8)


class EmuAug(EmuBackend):
    """b200seg_augment2d restated in numpy from the packed entries, plus the staging entry points"""

    def __init__(self):
        self.calls = []

    def augment2d_workspace(self, out_bytes, device):
        return torch.empty(max(int(out_bytes), 16), dtype=torch.uint8, device=device)

    def augment2d(self, src, params, n, max_hw, stages, out, msrc=None, mout=None, ws=None):
        raw = params.cpu().numpy().tobytes()
        s = src.cpu().numpy()
        ms = None if msrc is None else msrc.cpu().numpy()
        entries = [unpack(raw[i * AUG2D_PARAM_BYTES:(i + 1) * AUG2D_PARAM_BYTES]) for i in range(n)]
        self.calls.append(entries)
        for e in entries:
            h, w, c, f = e["h"], e["w"], e["c"], e["flags"]
            assert h * w <= max_hw and f & ~stages == 0
            img = s[e["src"]:e["src"] + h * w * c].reshape(h, w, c)
            img = oa.flip(img, f & 1, f & 2)
            mask = None
            if e["msrc"] >= 0 and ms is not None:
                mask = oa.flip(ms[e["msrc"]:e["msrc"] + h * w].reshape(h, w), f & 1, f & 2)
            if f & 4:
                img = emu_blur(img, e)
            if f & 8:
                img = emu_warp(img, e["minv"], False)
                mask = None if mask is None else emu_warp(mask, e["minv"], True)
            if f & 16:
                img = e["lut"][img]
            out[e["dst"]:e["dst"] + h * w * c].copy_(torch.from_numpy(np.ascontiguousarray(img).reshape(-1)))
            if mask is not None:
                mout[e["mdst"]:e["mdst"] + h * w].copy_(torch.from_numpy(np.ascontiguousarray(mask).reshape(-1)))

    def resize_linear(self, src, desc, out):
        s, d = src.cpu().numpy(), desc.cpu().numpy()
        for n in range(out.shape[0]):
            off, hw = int(d[n, 0]), int(d[n, 1])
            h, w = hw & 0xFFFFFFFF, hw >> 32
            out[n].copy_(torch.from_numpy(RZ.resize_u8(s[off:off + h * w].reshape(h, w), (out.shape[2], out.shape[1]))))


@pytest.fixture
def emu():
    be = EmuAug()
    runtime._set_backend_for_testing(be)
    yield be
    runtime._set_backend_for_testing(None)


def entry_for_case(case, src):
    """one fixture case -> a draw dict that runs exactly that stage"""
    d = {"hflip": False, "vflip": False, "blur": None, "kernel": None, "ssr": None, "bc": None}
    st = case["stage"]
    if st == "flip":
        d["hflip"], d["vflip"] = bool(case["hflip"]), bool(case["vflip"])
    elif st == "motion":
        d["blur"], d["kernel"] = "motion", np.array(case["kernel"], dtype=np.float32)
    elif st in ("median", "box"):
        d["blur"] = st
    elif st in ("warp", "warp_mask"):
        d["ssr"] = tuple(case["ssr"])
    else:
        d["bc"] = (case["alpha"], case["beta"])
    return d


def test_emulated_kernel_rule_equals_every_fixture(emu):
    """the packed table and the kernel's stated rule reproduce cv2 on every fixture case"""
    for i, case in enumerate(META):
        src = fixture_source(case)
        d = entry_for_case(case, src)
        h, w = src.shape[:2]
        c = 1 if src.ndim == 2 else 3
        flat = torch.from_numpy(src.reshape(-1).copy())
        if case["stage"] == "warp_mask":
            e, f = A2.param_entry(d, h, w, 1, 0, 0, 0, 0)
            out, mout = torch.zeros(h * w, dtype=torch.uint8), torch.zeros(h * w, dtype=torch.uint8)
            A2.launch(emu, flat, [(e, f, h * w)], out, msrc=flat.clone(), mout=mout)
            got = mout
        else:
            e, f = A2.param_entry(d, h, w, c, 0, 0)
            got = torch.zeros(h * w * c, dtype=torch.uint8)
            A2.launch(emu, flat, [(e, f, h * w)], got)
        assert matches_fixture(i, got.numpy().reshape(src.shape)), (i, case)


def test_transform_compose_is_the_oracle(emu):
    rng = np.random.RandomState(0)
    aug = b200.Segmenation_Aug()
    for seed in range(60):
        h, w = (int(v) for v in rng.randint(1, 40, 2))
        img = rng.randint(0, 256, (h, w, 3) if seed % 2 else (h, w)).astype(np.uint8)
        mask = (rng.rand(h, w) > 0.5).astype(np.uint8) * 255
        random.seed(seed)
        got = aug.transform_compose(image=img, mask=mask)
        random.seed(seed)
        want_img, want_mask = oa.compose(img, mask)
        assert np.array_equal(got["image"], want_img) and np.array_equal(got["mask"], want_mask), seed


def test_data_augmentation_writes_the_oracle_files(emu, tmp_path):
    rng = np.random.RandomState(1)
    rows = []
    for r, (h, w) in enumerate(((21, 34), (17, 9))):
        ip, mp = str(tmp_path / f"img{r}.png"), str(tmp_path / f"mask{r}.png")
        cv2.imwrite(ip, rng.randint(0, 256, (h, w, 3)).astype(np.uint8))
        cv2.imwrite(mp, (rng.rand(h, w) > 0.5).astype(np.uint8) * 255)
        rows.append((ip, mp))
    csv = tmp_path / "train.csv"
    csv.write_text("Image,Mask\n" + "".join(f"{a},{b}\n" for a, b in rows))
    for sub in ("got", "want"):
        os.makedirs(tmp_path / sub / "Image")
        os.makedirs(tmp_path / sub / "Mask")
    random.seed(7)
    b200.Segmenation_Aug().DataAugmentation(str(csv), 12, str(tmp_path / "got"))
    assert len(emu.calls) == 2 and len(emu.calls[0]) == 12          # one launch per row
    random.seed(7)
    for index, (ip, mp) in enumerate(rows):                            # the reference's loop, with the oracle
        src_image, src_mask = cv2.imread(ip), cv2.imread(mp, 0)
        for i in range(12):
            image, mask = oa.compose(src_image, src_mask)
            cv2.imwrite(str(tmp_path / "want" / "Image" / f"{index}_{i}.bmp"), image)
            cv2.imwrite(str(tmp_path / "want" / "Mask" / f"{index}_{i}.bmp"), mask)
    for sub in ("Image", "Mask"):
        names = sorted(os.listdir(tmp_path / "want" / sub))
        assert names == sorted(os.listdir(tmp_path / "got" / sub)) and len(names) == 24
        for nm in names:
            assert (tmp_path / "want" / sub / nm).read_bytes() == (tmp_path / "got" / sub / nm).read_bytes(), nm


def test_transform_batch_gray_is_the_bgr_file_path(emu):
    rng = np.random.RandomState(2)
    imgs = rng.randint(0, 256, (40, 13, 18)).astype(np.uint8)
    masks = (rng.rand(40, 13, 18) > 0.5).astype(np.uint8)
    random.seed(11)
    x, y = b200.Segmenation_Aug().transform_batch(torch.from_numpy(imgs), torch.from_numpy(masks))
    random.seed(11)
    for i in range(40):
        d = oa.draw()
        assert np.array_equal(x[i].numpy(), oa.as_bgr_gray(imgs[i], d)), i
        assert np.array_equal(y[i].numpy(), oa.apply(d, imgs[i], masks[i])[1]), i


def test_stager_augment_is_oracle_then_resize_then_zscore(emu):
    rng = np.random.RandomState(3)
    sizes = [(30, 41), (17, 17), (64, 9), (5, 70)]
    imgs = [rng.randint(0, 256, s).astype(np.uint8) for s in sizes]
    labs = [(rng.rand(*s) > 0.6).astype(np.uint8) * 255 for s in sizes]
    st = b200.InputStager("cpu", (4, 24, 24), backend=emu, max_source_pixels=4096, augment=b200.Segmenation_Aug())
    for with_labels in (True, False):
        random.seed(5)
        st.put(imgs, labs if with_labels else None)
        x, y = st.get()
        random.seed(5)
        ai, al = [], []
        for im, lb in zip(imgs, labs):
            d = oa.draw()
            ai.append(oa.as_bgr_gray(im, d))
            al.append(oa.apply(d, im, lb)[1])
        assert torch.equal(x, OS.zscore_u8(RZ.resize_u8_batch(ai, (24, 24))))
        if with_labels:
            assert torch.equal(y, OS.labels_from_u8(RZ.resize_u8_batch(al, (24, 24))))
        else:
            assert y is None
    with pytest.raises(ValueError):
        st.put(imgs, [lb[:, :-1] for lb in labs])
