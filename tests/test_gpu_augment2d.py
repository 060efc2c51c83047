"""2-D augmentation (Segmenation_Aug, csrc/augment2d.cu) on the GPU: every cv2 fixture byte for byte in one ragged
launch per stage, ``transform_compose`` / ``transform_batch`` / ``DataAugmentation``'s batches against the cv2 oracle
for the same seed, the gray per-step form against the BGR file path, ``InputStager(augment=...)`` against oracle ->
cv2.resize -> z-score, bit-identical reruns and guard bands around the outputs."""
import json
import os
import random

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
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

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


DEV = torch.device("cuda", 0)
GUARD = 64


def case_draw(case):
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


def run_ragged(items, masks=False):
    """[(draw, numpy image)] -> outputs of one launch; sources packed back to back, outputs inside guard bands.
    masks: the items are masks (c = 1) and go through the mask path (nearest warp, no blur, no table)"""
    srcs, entries, outs, soff, doff = [], [], [], 0, GUARD
    for d, img in items:
        h, w = img.shape[:2]
        c = 1 if img.ndim == 2 else 3
        if masks:
            e, f = A2.param_entry(d, h, w, 1, soff, doff, soff, doff)
        else:
            e, f = A2.param_entry(d, h, w, c, soff, doff)
        entries.append((e, f, h * w))
        srcs.append(img.reshape(-1))
        outs.append((doff, img.shape))
        soff += img.size
        doff += img.size + GUARD
    src = torch.from_numpy(np.concatenate(srcs)).to(DEV)
    out = torch.full((doff,), 0xA5, dtype=torch.uint8, device=DEV)
    be = runtime.get_backend(src)
    if masks:
        img_out = torch.full((doff,), 0xA5, dtype=torch.uint8, device=DEV)
        A2.launch(be, src, entries, img_out, msrc=src, mout=out)
    else:
        A2.launch(be, src, entries, out)
    o = out.cpu().numpy()
    gaps = np.ones(doff, bool)
    res = []
    for off, shape in outs:
        n = int(np.prod(shape))
        res.append(o[off:off + n].reshape(shape))
        gaps[off:off + n] = False
    assert (o[gaps] == 0xA5).all(), "a write outside the outputs"
    return res, entries, src, be


@pytest.mark.parametrize("stage", ["flip", "motion", "median", "box", "warp", "warp_mask", "lut"])
def test_every_fixture_byte_for_byte(stage):
    idx = [i for i, c in enumerate(META) if c["stage"] == stage]
    items = [(case_draw(META[i]), fixture_source(META[i])) for i in idx]
    got, _, _, _ = run_ragged(items, masks=stage == "warp_mask")
    for i, g in zip(idx, got):
        assert matches_fixture(i, g), (i, META[i])


def test_transform_compose_equals_the_oracle_on_mixed_batches():
    rng = np.random.RandomState(0)
    aug = b200.Segmenation_Aug()
    stages = set()
    for seed in range(120):
        h, w = ((512, 512) if seed % 10 == 0 else tuple(int(v) for v in rng.randint(1, 90, 2)))
        img = rng.randint(0, 256, (h, w, 3) if seed % 2 else (h, w)).astype(np.uint8)
        mask = (rng.rand(h, w) > 0.5).astype(np.uint8)
        random.seed(seed)
        d = oa.draw()
        stages.add((d["blur"], d["ssr"] is not None, d["bc"] is not None))
        random.seed(seed)
        got = aug.transform_compose(image=img, mask=mask)
        want_img, want_mask = oa.apply(d, img, mask)
        assert np.array_equal(got["image"], want_img) and np.array_equal(got["mask"], want_mask), seed
    assert len({s[0] for s in stages}) == 4


def test_many_copies_of_one_source_in_one_launch():
    """DataAugmentation's batch: every entry reads the same uploaded source"""
    rng = np.random.RandomState(1)
    img = rng.randint(0, 256, (61, 47, 3)).astype(np.uint8)
    mask = (rng.rand(61, 47) > 0.5).astype(np.uint8) * 255
    random.seed(3)
    draws = [A2.draw_params() for _ in range(400)]
    images, masks = A2.Segmenation_Aug._run_copies(img, mask, draws, filter_cn=3)
    assert {d["blur"] for d in draws} == {None, "motion", "median", "box"}
    for i, d in enumerate(draws):
        wi, wm = oa.apply(d, img, mask)
        assert np.array_equal(images[i], wi) and np.array_equal(masks[i], wm), i


@pytest.mark.parametrize("shape", [(8, 512, 512), (6, 37, 53), (5, 9, 1)])
def test_transform_batch_equals_the_oracle_and_the_bgr_file_path(shape):
    rng = np.random.RandomState(2)
    imgs = rng.randint(0, 256, shape).astype(np.uint8)
    masks = (rng.rand(*shape) > 0.5).astype(np.uint8)
    aug = b200.Segmenation_Aug()
    for seed in range(6):
        random.seed(seed)
        x, y = aug.transform_batch(torch.from_numpy(imgs).to(DEV), torch.from_numpy(masks).to(DEV))
        random.seed(seed)
        xb, yb = aug.transform_batch(torch.from_numpy(np.repeat(imgs[..., None], 3, axis=3)).to(DEV),
                                     torch.from_numpy(masks).to(DEV))
        assert torch.equal(x, xb[..., 0]) and torch.equal(y, yb)       # gray = channel 0 of gray-valued BGR
        random.seed(seed)
        for i in range(shape[0]):
            d = oa.draw()
            assert np.array_equal(x[i].cpu().numpy(), oa.as_bgr_gray(imgs[i], d)), (seed, i)
            assert np.array_equal(y[i].cpu().numpy(), oa.apply(d, imgs[i], masks[i])[1]), (seed, i)
            wb = oa.apply(d, np.repeat(imgs[i][..., None], 3, axis=2))[0]
            assert np.array_equal(xb[i].cpu().numpy(), wb), (seed, i)


def test_stager_augment_equals_oracle_resize_zscore():
    rng = np.random.RandomState(4)
    sizes = [(1000, 700), (700, 1000), (512, 512), (333, 517), (1, 9), (64, 1), (999, 701), (256, 300)]
    imgs = [rng.randint(0, 256, s).astype(np.uint8) for s in sizes]
    labs = [(rng.rand(*s) > 0.7).astype(np.uint8) for s in sizes]
    st = b200.InputStager(DEV, (8, 512, 512), max_source_pixels=4 << 20, augment=b200.Segmenation_Aug())
    for rep in range(3):
        random.seed(rep)
        st.put(imgs, labs)
        x, y = st.get()
        torch.cuda.synchronize()
        random.seed(rep)
        ai, al = [], []
        for im, lb in zip(imgs, labs):
            d = oa.draw()
            ai.append(oa.as_bgr_gray(im, d))
            al.append(oa.apply(d, im, lb)[1])
        assert torch.equal(x.cpu(), OS.zscore_u8(RZ.resize_u8_batch(ai, (512, 512))))
        assert torch.equal(y.cpu(), OS.labels_from_u8(RZ.resize_u8_batch(al, (512, 512))))
        st.release()


def test_reruns_are_bit_identical():
    rng = np.random.RandomState(5)
    items = []
    random.seed(9)
    for i in range(64):
        h, w = (int(v) for v in rng.randint(1, 200, 2))
        items.append((A2.draw_params(), rng.randint(0, 256, (h, w, 3) if i % 2 else (h, w)).astype(np.uint8)))
    a, entries, src, be = run_ragged(items)
    b, _, _, _ = run_ragged(items)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    flags = 0
    for _, f, _ in entries:
        flags |= f
    assert flags == 31
