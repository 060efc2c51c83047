"""2-D image resize kernel (csrc/resize2d.cu) on the GPU: byte-equal to cv2's fixtures and to the numpy restatement
(oracle/resize2d.py) in both output modes, ragged launches with a 4096^2 source, guard bands, bit-identical reruns,
the stager's resize mode against the reference's dataset fixtures, and inference2d end to end against the oracle chain
around the existing predict_mask."""
import os

import numpy as np
import pytest
import torch

from oracle import nets as onets
from oracle import resnet as ores
from oracle import resize2d as RZ
from oracle import staging as OS
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import inference as inf
from pytorchdeeplearing_b200 import runtime
from conftest import GOLDEN

pytestmark = pytest.mark.gpu
GOLD = dict(np.load(os.path.join(GOLDEN, "resize2d.npz")))
CASES = [str(c) for c in GOLD["rs_cases"]]
GUARD = 4096


@pytest.fixture(autouse=True)
def _restore_precision():
    prev = b200.get_precision()
    yield
    b200.set_precision(prev)


def be():
    return runtime.cuda_backend()


def run(images, dsize, dtype=torch.uint8, shift=0):
    """one launch over the ragged list ``images`` into a guarded (N, oH, oW) buffer; ``shift`` elements of offset make
    the output rows unaligned"""
    ow, oh = dsize
    pix = torch.from_numpy(np.concatenate([np.ascontiguousarray(im).ravel() for im in images])).cuda()
    offs = np.cumsum([0] + [im.size for im in images])[:-1]
    desc = inf.resize_desc(be(), [(o, im.shape[0], im.shape[1]) for o, im in zip(offs, images)], pix.device)
    n = len(images) * oh * ow
    fill = 0xAB if dtype == torch.uint8 else float("nan")
    buf = torch.full((n + 2 * GUARD + shift,), fill, dtype=dtype, device="cuda")
    out = buf[GUARD + shift:GUARD + shift + n].view(len(images), oh, ow)
    be().resize_linear(pix, desc, out)
    torch.cuda.synchronize()
    g = torch.cat([buf[:GUARD + shift], buf[GUARD + shift + n:]]).cpu()
    assert bool((g == fill).all()) if dtype == torch.uint8 else bool(torch.isnan(g).all()), "guard band overwritten"
    return out.cpu().numpy()


def same_f32(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.int32), np.asarray(b, np.float32).view(np.int32))


@pytest.mark.parametrize("case", CASES)
def test_kernel_equals_cv2_fixture_in_both_modes(case):
    src, dsize, dst = GOLD[f"rs_{case}_src"], tuple(int(v) for v in GOLD[f"rs_{case}_dsize"]), GOLD[f"rs_{case}_dst"]
    assert np.array_equal(run([src], dsize)[0], dst)
    assert same_f32(run([src], dsize, torch.float32)[0], RZ.to_unit_float(dst))
    assert np.array_equal(run([src], dsize, shift=1)[0], dst)                       # unaligned rows: scalar stores


@pytest.mark.parametrize("case", ["square", "nonsquare", "resnet"])
def test_kernel_reproduces_the_reference_inference_lines(case):
    image, new_size = GOLD[f"inf_{case}_image"], tuple(int(v) for v in GOLD[f"inf_{case}_newsize"])
    assert same_f32(run([image], new_size, torch.float32), GOLD[f"inf_{case}_x"])
    if case != "resnet":
        assert np.array_equal(run([GOLD[f"inf_{case}_mask"]], image.shape)[0], GOLD[f"inf_{case}_out"])


def test_kernel_against_the_oracle_on_a_seeded_sweep():
    rng = np.random.RandomState(99)
    for t in range(240):
        h, w, oh, ow = (int(v) for v in rng.randint(1, 600, 4))
        if t % 6 == 0:
            oh, ow = max(1, h // 2), max(1, w // 2)
        elif t % 6 == 1:
            oh, ow = max(1, h // 4), max(1, w // 4)
        kind = t % 3
        img = (rng.randint(0, 256, (h, w)) if kind == 0 else
               (rng.rand(h, w) > 0.5) * 255 if kind == 1 else rng.randint(0, 4, (h, w))).astype(np.uint8)
        want = RZ.resize_u8(img, (ow, oh))
        got = run([img], (ow, oh), shift=t % 2)[0]
        assert np.array_equal(got, want), (h, w, oh, ow, kind)
        assert same_f32(run([img], (ow, oh), torch.float32)[0], RZ.to_unit_float(want)), (h, w, oh, ow, kind)


@pytest.mark.parametrize("dsize", [(512, 512), (509, 383)])
def test_one_ragged_launch_equals_per_sample_results(dsize):
    rng = np.random.RandomState(3)
    sizes = [(4096, 4096), (1, 1), (300, 417), (777, 33), (512, 512), (1, 700)]
    images = [rng.randint(0, 256, s).astype(np.uint8) for s in sizes]
    for dtype in (torch.uint8, torch.float32):
        got = run(images, dsize, dtype)
        for i, im in enumerate(images):
            alone = run([im], dsize, dtype)[0]
            want = RZ.resize_u8(im, dsize)
            assert np.array_equal(got[i], alone), (i, dtype)
            assert np.array_equal(got[i], want if dtype == torch.uint8 else RZ.to_unit_float(want)), (i, dtype)


def test_reruns_are_bit_identical():
    rng = np.random.RandomState(5)
    images = [rng.randint(0, 256, s).astype(np.uint8) for s in [(1024, 1024), (300, 417), (5, 3)]]
    for dtype in (torch.uint8, torch.float32):
        a, b = run(images, (512, 512), dtype), run(images, (512, 512), dtype)
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_argument_checks():
    pix = torch.zeros(16, dtype=torch.uint8, device="cuda")
    desc = inf.resize_desc(be(), [(0, 4, 4)], pix.device)
    dev = torch.cuda.current_device()

    def call(n, mode):
        be()._check(be().lib.b200seg_resize_linear_u8(pix.data_ptr(), desc.data_ptr(), n, 4, 4, pix.data_ptr(), mode,
                                                      dev, torch.cuda.current_stream().cuda_stream))

    with pytest.raises(RuntimeError, match="out_mode"):
        call(1, 99)
    with pytest.raises(RuntimeError, match="sizes"):
        call(0, 17)
    with pytest.raises(ValueError, match="resize batch"):
        inf.resize_desc(be(), [], pix.device)
    with pytest.raises(TypeError):
        b200.resize2d(np.zeros((4, 4), np.float32), (2, 2))
    t = b200.resize2d(torch.from_numpy(GOLD["rs_down2_src"]).cuda(), (100, 128))
    assert t.is_cuda and np.array_equal(t.cpu().numpy(), GOLD["rs_down2_dst"])
    assert np.array_equal(b200.resize2d(GOLD["rs_nonsquare_src"], (64, 96)), GOLD["rs_nonsquare_dst"])


# ---------------------------------------------------------------------------------------------- input staging
def fixture_images(prefix):
    n = sum(1 for k in GOLD if k.startswith(prefix + "_img"))
    return [GOLD[f"{prefix}_img{i}"] for i in range(n)], [GOLD.get(f"{prefix}_lab{i}") for i in range(n)]


def test_stager_resize_mode_reproduces_the_segmentation_dataset():
    imgs, labs = fixture_images("seg")
    st = b200.InputStager("cuda", (len(imgs), 64, 64), max_source_pixels=sum(im.size for im in imgs))
    for _ in range(3):                                  # reuse both slots
        st.put(imgs, labs)
        x, y = st.get()
        st.release()
        torch.cuda.synchronize()
        assert same_f32(x.cpu().numpy(), GOLD["seg_x"])
        assert np.array_equal(y.cpu().numpy(), GOLD["seg_y"])


def test_stager_resize_mode_reproduces_the_classification_dataset():
    imgs, _ = fixture_images("cls")
    st = b200.InputStager("cuda", (len(imgs), 48, 48), max_source_pixels=sum(im.size for im in imgs))
    st.put(imgs)
    x, y = st.get()
    torch.cuda.synchronize()
    assert y is None and same_f32(x.cpu().numpy(), GOLD["cls_x"])


def test_stager_resize_mode_at_the_target_size_equals_the_plain_path():
    rng = np.random.RandomState(8)
    imgs = rng.randint(0, 256, (4, 96, 128)).astype(np.uint8)
    labs = (rng.rand(4, 96, 128) > 0.6).astype(np.uint8) * 3
    plain = b200.InputStager("cuda", (4, 96, 128))
    ragged = b200.InputStager("cuda", (4, 96, 128), max_source_pixels=imgs.size)
    plain.put(imgs, labs)
    ragged.put(list(imgs), list(labs))
    (xa, ya), (xb, yb) = plain.get(), ragged.get()
    torch.cuda.synchronize()
    assert torch.equal(xa.view(torch.int32), xb.view(torch.int32)) and torch.equal(ya, yb)
    # a non-square target: cv2.resize(img, (W, H)) then the z-score
    src = [rng.randint(0, 256, s).astype(np.uint8) for s in [(200, 100), (31, 517), (96, 128), (7, 9)]]
    ragged.put(src)
    x, _ = ragged.get()
    torch.cuda.synchronize()
    want = OS.zscore_u8(RZ.resize_u8_batch(src, (128, 96))).numpy()
    assert same_f32(x.cpu().numpy(), want)


# ---------------------------------------------------------------------------------------------- inference2d
def seeded(kind, ncls, seed=0):
    if kind == "vnet":
        model, spec = b200.VNet2d(1, ncls), onets.vnet3d_state_spec(1, ncls, dims=2)
    elif kind == "unet":
        model, spec = b200.UNet2d(1, ncls), onets.unet_state_spec(1, ncls, 2)
    else:
        model, spec = b200.ResNet2d(1, ncls), ores.resnet_state_spec(1, ncls, 2)
    model.load_state_dict(onets.init_state_dict(spec, seed=seed, randomize_affine=True))
    return model.cuda().eval()


def oracle_input(img, new_size):
    return torch.from_numpy(RZ.to_unit_float(RZ.resize_u8(img, new_size)))[None, None].cuda()


@pytest.mark.parametrize("kind", ["vnet", "unet"])
@pytest.mark.parametrize("ncls", [1, 3])
@pytest.mark.parametrize("shape,new_size", [((300, 300), (128, 128)), ((237, 410), (160, 96))])
def test_inference2d_segmenters_equal_the_oracle_chain(kind, ncls, shape, new_size):
    b200.set_precision("fp32")
    model = seeded(kind, ncls)
    img = np.random.RandomState(11).randint(0, 256, shape).astype(np.uint8)
    got = b200.inference2d(model, img, new_size)
    m = b200.predict_mask(model, oracle_input(img, new_size))[0].cpu().numpy()
    want = RZ.resize_u8(m, img.shape)
    assert got.dtype == np.uint8 and got.shape == (shape[1], shape[0]) and np.array_equal(got, want)


@pytest.mark.parametrize("ncls", [1, 4])
def test_inference2d_resnet_equals_the_classifier_predict(ncls):
    b200.set_precision("fp32")
    model = seeded("resnet", ncls, seed=3)
    for seed in range(3):
        img = np.random.RandomState(seed).randint(0, 256, (150, 210)).astype(np.uint8)
        got = b200.inference2d(model, img, (64, 48))
        with torch.no_grad():
            logits = model(oracle_input(img, (64, 48)))[0].float().cpu()
        if ncls == 1:
            want = int(torch.sigmoid(logits[0]) > 0.5) * 255
        else:
            want = int(np.argmax(torch.softmax(logits, 0).numpy()))
        assert isinstance(got, np.int64) and got == want


def test_inference2d_device_chain_does_not_synchronise():
    b200.set_precision("bf16")
    model = seeded("unet", 1)
    src = torch.from_numpy(np.random.RandomState(2).randint(0, 256, (333, 271)).astype(np.uint8)).cuda()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m = inf._inference2d_device(model, src, (128, 128), 0.5)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert tuple(m.shape) == (271, 333)
