"""2-D image resize (cv2.resize INTER_LINEAR, reference model/dataset.py:63,140,154 and the 2-D ``inference`` methods)
without a GPU: the numpy restatement (oracle/resize2d.py) against fixtures recorded from cv2 and the reference's own
dataset classes and ``inference`` lines, a seeded sweep against cv2 itself where it imports, and the Python layer
(``resize2d``, ``inference2d``, ``InputStager(max_source_pixels=...)``) on an emulated backend."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import nets as onets
from oracle import resnet as ores
from oracle import resize2d as RZ
from oracle import staging as OS
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import runtime
from conftest import GOLDEN
from emu_backend import EmuBackend

GOLD = dict(np.load(os.path.join(GOLDEN, "resize2d.npz")))
CASES = [str(c) for c in GOLD["rs_cases"]]


def seg_inputs(prefix):
    n = sum(1 for k in GOLD if k.startswith(prefix + "_img"))
    return [GOLD[f"{prefix}_img{i}"] for i in range(n)], [GOLD.get(f"{prefix}_lab{i}") for i in range(n)]


@pytest.mark.parametrize("case", CASES)
def test_oracle_equals_cv2_on_every_fixture_case(case):
    src, dsize, dst = GOLD[f"rs_{case}_src"], tuple(GOLD[f"rs_{case}_dsize"]), GOLD[f"rs_{case}_dst"]
    out = RZ.resize_u8(src, dsize)
    assert out.dtype == np.uint8 and out.shape == dst.shape == (dsize[1], dsize[0])
    assert np.array_equal(out, dst)


def test_fixture_cases_cover_the_issue_list():
    shapes = {c: (GOLD[f"rs_{c}_src"].shape, tuple(GOLD[f"rs_{c}_dsize"])) for c in CASES}
    assert shapes["src1x1"][0] == (1, 1) and shapes["src1x700"][0] == (1, 700) and shapes["dst1x1"][1] == (1, 1)
    assert shapes["identity"][0] == tuple(reversed(shapes["identity"][1]))
    assert shapes["down2"][0] == (256, 200) and shapes["down2"][1] == (100, 128)
    assert shapes["down4"][0] == (256, 256) and shapes["down4"][1] == (64, 64)
    assert set(np.unique(GOLD["rs_binary_down_src"])) == {0, 255}
    assert set(np.unique(GOLD["rs_labels_up_src"])) == {0, 1, 2, 3}


def test_oracle_and_staging_reproduce_the_segmentation_dataset():
    imgs, labs = seg_inputs("seg")
    assert any(im.shape != (64, 64) for im in imgs)
    x = OS.zscore_u8(RZ.resize_u8_batch(imgs, (64, 64)))
    y = OS.labels_from_u8(RZ.resize_u8_batch(labs, (64, 64)))
    assert np.array_equal(x.numpy().view(np.int32), GOLD["seg_x"].view(np.int32))
    assert np.array_equal(y.numpy(), GOLD["seg_y"])


def test_oracle_and_staging_reproduce_the_classification_dataset():
    imgs, _ = seg_inputs("cls")
    x = OS.zscore_u8(RZ.resize_u8_batch(imgs, (48, 48)))
    assert np.array_equal(x.numpy().view(np.int32), GOLD["cls_x"].view(np.int32))


@pytest.mark.parametrize("case", ["square", "nonsquare", "resnet"])
def test_oracle_reproduces_the_inference_lines(case):
    image, new_size = GOLD[f"inf_{case}_image"], tuple(GOLD[f"inf_{case}_newsize"])
    x = RZ.to_unit_float(RZ.resize_u8(image, new_size))
    assert np.array_equal(x[None].view(np.int32), GOLD[f"inf_{case}_x"].view(np.int32))
    if case != "resnet":
        out = RZ.resize_u8(GOLD[f"inf_{case}_mask"], image.shape)
        assert out.shape == tuple(reversed(image.shape))
        assert np.array_equal(out, GOLD[f"inf_{case}_out"])


def test_oracle_against_cv2_on_a_seeded_sweep():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.RandomState(1234)
    pairs = 0
    for _ in range(220):
        h, w, oh, ow = (int(v) for v in rng.randint(1, 700, 4))
        if rng.rand() < 0.2:
            oh, ow = max(1, h // 2), max(1, w // 2)
        kind = rng.randint(3)
        img = (rng.randint(0, 256, (h, w)) if kind == 0 else
               (rng.rand(h, w) > 0.5) * 255 if kind == 1 else rng.randint(0, 4, (h, w))).astype(np.uint8)
        assert np.array_equal(RZ.resize_u8(img, (ow, oh)), cv2.resize(img, (ow, oh))), (h, w, oh, ow, kind)
        pairs += 1
    assert pairs >= 200


# ---------------------------------------------------------------------------------------------- emulated backend
class EmuResize(EmuBackend):
    """the resize entry point through the oracle, plus what inference2d uses around it"""

    def __init__(self):
        self.resize_calls = []

    def upload_bytes(self, raw, device):
        pad = (len(raw) + 15) // 16 * 16
        return torch.frombuffer(bytearray(raw.ljust(pad, b"\0")), dtype=torch.uint8).to(device)

    def resize_linear(self, src, desc, out):
        assert src.dtype == torch.uint8 and desc.dtype == torch.int64 and tuple(desc.shape) == (out.shape[0], 2)
        s, d = src.cpu().numpy(), desc.cpu().numpy()
        self.resize_calls.append(d.copy())
        for n in range(out.shape[0]):
            off, hw = int(d[n, 0]), int(d[n, 1])
            h, w = hw & 0xFFFFFFFF, hw >> 32
            v = RZ.resize_u8(s[off:off + h * w].reshape(h, w), (out.shape[2], out.shape[1]))
            out[n].copy_(torch.from_numpy(v if out.dtype == torch.uint8 else RZ.to_unit_float(v)))

    def cls_head_fwd(self, x, w1, b1, w2, b2, pooled, hidden, logits):
        p = x.float().reshape(x.shape[0], -1, x.shape[-1]).mean(1)
        h = F.relu(F.linear(p, w1, b1))
        pooled.copy_(p)
        hidden.copy_(h)
        logits.copy_(F.linear(h, w2, b2))


@pytest.fixture
def emu():
    be = EmuResize()
    runtime._set_backend_for_testing(be)
    prev = b200.get_precision()
    b200.set_precision("fp32")
    yield be
    b200.set_precision(prev)
    runtime._set_backend_for_testing(None)


def image(shape, seed=0):
    return np.random.RandomState(seed).randint(0, 256, size=shape).astype(np.uint8)


def test_resize2d_arrays_tensors_and_batches(emu):
    a = image((37, 53))
    out = b200.resize2d(a, (40, 30), device="cpu")
    assert isinstance(out, np.ndarray) and out.shape == (30, 40) and np.array_equal(out, RZ.resize_u8(a, (40, 30)))
    batch = np.stack([a, image((37, 53), 1)])
    t = b200.resize2d(torch.from_numpy(batch), (16, 64))
    assert isinstance(t, torch.Tensor) and tuple(t.shape) == (2, 64, 16) and t.dtype == torch.uint8
    for i in range(2):
        assert np.array_equal(t[i].numpy(), RZ.resize_u8(batch[i], (16, 64)))
    # one launch with one descriptor per sample
    off, hw = emu.resize_calls[-1][:, 0].tolist(), emu.resize_calls[-1][:, 1].tolist()
    assert off == [0, 37 * 53] and hw == [37 | (53 << 32)] * 2


def test_resize2d_refusals(emu):
    with pytest.raises(TypeError, match="uint8"):
        b200.resize2d(np.zeros((4, 4), np.float32), (2, 2), device="cpu")
    with pytest.raises(TypeError, match="uint8"):
        b200.resize2d(torch.zeros((4, 4), dtype=torch.int16), (2, 2))
    with pytest.raises(ValueError, match="shape"):
        b200.resize2d(np.zeros((4,), np.uint8), (2, 2), device="cpu")
    with pytest.raises(ValueError, match="shape"):
        b200.resize2d(np.zeros((1, 2, 4, 4), np.uint8), (2, 2), device="cpu")
    with pytest.raises(ValueError, match=">= 1"):
        b200.resize2d(np.zeros((0, 4), np.uint8), (2, 2), device="cpu")
    for bad in ((0, 2), (2,), (2, 2, 2)):
        with pytest.raises(ValueError, match="dsize"):
            b200.resize2d(np.zeros((4, 4), np.uint8), bad, device="cpu")


def seeded(kind, ncls, seed=0):
    if kind == "vnet":
        model = b200.VNet2d(1, ncls)
        spec = onets.vnet3d_state_spec(1, ncls, dims=2)
    elif kind == "unet":
        model = b200.UNet2d(1, ncls)
        spec = onets.unet_state_spec(1, ncls, 2)
    else:
        model = b200.ResNet2d(1, ncls)
        spec = ores.resnet_state_spec(1, ncls, 2)
    model.load_state_dict(onets.init_state_dict(spec, seed=seed, randomize_affine=True))
    return model.eval()


def oracle_chain(model, img, new_size, thr=0.5):
    x = torch.from_numpy(RZ.to_unit_float(RZ.resize_u8(img, new_size)))[None, None]
    m = b200.predict_mask(model, x, thr)[0].numpy()
    return RZ.resize_u8(m, img.shape)


@pytest.mark.parametrize("kind,ncls", [("vnet", 1), ("unet", 3)])
def test_inference2d_is_the_oracle_chain(emu, kind, ncls):
    model = seeded(kind, ncls)
    img = image((50, 41), seed=2)
    got = b200.inference2d(model, img, (32, 32))
    assert got.dtype == np.uint8 and got.shape == (41, 50)         # cv2.resize(mask, image.shape): (W, H)
    assert np.array_equal(got, oracle_chain(model, img, (32, 32)))


def test_inference2d_non_square_network_input(emu):
    model = seeded("unet", 1)
    img = image((30, 70), seed=3)
    got = b200.inference2d(model, img, (48, 32), out_threshold=0.3)
    assert got.shape == (70, 30) and np.array_equal(got, oracle_chain(model, img, (48, 32), 0.3))
    # the network saw cv2.resize(image, (48, 32)) / 255: a (32, 48) input
    assert emu.resize_calls[-2][0, 1] == 30 | (70 << 32)


@pytest.mark.parametrize("ncls", [1, 3])
def test_inference2d_resnet_returns_the_classifier_prediction(emu, ncls):
    model = seeded("resnet", ncls, seed=5)
    img = image((45, 60), seed=4)
    got = b200.inference2d(model, img, (32, 32))
    x = torch.from_numpy(RZ.to_unit_float(RZ.resize_u8(img, (32, 32))))[None, None]
    with torch.no_grad():
        logits = model(x)[0]
    want = (int(torch.sigmoid(logits[0]) > 0.5) * 255) if ncls == 1 else int(torch.softmax(logits, 0).argmax())
    assert isinstance(got, np.int64) and got == want


def test_inference2d_refusals(emu):
    img = image((20, 20))
    with pytest.raises(ValueError, match="3-D"):
        b200.inference2d(b200.VNet3d(1, 2), img)
    with pytest.raises(ValueError, match="3-D"):
        b200.inference2d(b200.ResNet3d(1, 2), img)
    model = seeded("unet", 1)
    with pytest.raises(TypeError, match="uint8"):
        b200.inference2d(model, img.astype(np.float32))
    with pytest.raises(ValueError, match=r"\(H, W\)"):
        b200.inference2d(model, img[None])
    with pytest.raises(ValueError, match="dsize"):
        b200.inference2d(model, img, (32,))
    # the existing predict paths keep their classifier TypeError
    with pytest.raises(TypeError, match="classifier"):
        b200.predict(seeded("resnet", 2), img[None].astype(np.float32))


def test_stager_resize_mode_packs_a_ragged_batch(emu):
    sizes = [(33, 70), (64, 64), (2, 3), (100, 7)]
    imgs = [image(s, i) for i, s in enumerate(sizes)]
    labs = [(image(s, 10 + i) > 150).astype(np.uint8) * (255 if i % 2 else 3) for i, s in enumerate(sizes)]
    st = InputStagerCPU((4, 32, 32), max_source_pixels=sum(h * w for h, w in sizes))
    st.put(imgs, labs)
    x, y = st.get()
    assert np.array_equal(x.numpy().view(np.int32),
                          OS.zscore_u8(RZ.resize_u8_batch(imgs, (32, 32))).numpy().view(np.int32))
    assert np.array_equal(y.numpy(), OS.labels_from_u8(RZ.resize_u8_batch(labs, (32, 32))).numpy())
    # the slot holds the image descriptors, the label descriptors, then the image pixels and the label pixels
    h = st._slots[0]["h_src"]
    table = h[:2 * 16 * 4].numpy().view(np.int64).reshape(8, 2)
    offs = np.cumsum([0] + [a * b for a, b in sizes + sizes])[:-1]
    assert table[:, 0].tolist() == offs.tolist()
    assert table[:, 1].tolist() == [a | (b << 32) for a, b in sizes + sizes]
    base = 2 * 16 * 4
    assert np.array_equal(h[base + offs[4]:base + offs[4] + 33 * 70].numpy(), labs[0].ravel())
    assert st._slots[0]["used"] == base + 2 * sum(a * b for a, b in sizes)


def InputStagerCPU(shape, **kw):
    return b200.InputStager("cpu", shape, backend=runtime.get_backend(torch.empty(0)), **kw)


def test_stager_resize_mode_non_square_target_and_no_labels(emu):
    imgs = [image((40, 90), 1), image((17, 23), 2)]
    st = InputStagerCPU((2, 16, 48), max_source_pixels=4000)
    st.put(imgs)
    x, y = st.get()
    assert y is None and tuple(x.shape) == (2, 1, 16, 48)
    want = OS.zscore_u8(np.stack([RZ.resize_u8(im, (48, 16)) for im in imgs]))      # cv2.resize(img, (W, H))
    assert np.array_equal(x.numpy().view(np.int32), want.numpy().view(np.int32))


def test_stager_resize_mode_refusals(emu):
    st = InputStagerCPU((2, 16, 16), max_source_pixels=1000)
    with pytest.raises(ValueError, match="max_source_pixels"):
        st.put([image((30, 31)), image((10, 10))])                                   # 930 + 100 > 1000
    with pytest.raises(ValueError, match="max_source_pixels"):
        st.put([image((20, 20)), image((10, 10))], [image((30, 31)), image((10, 10))])
    st.put([image((20, 20)), image((24, 25))])                                       # exactly 1000 fits
    st.get()
    with pytest.raises(ValueError, match="expected 2 images"):
        st.put([image((20, 20))])
    with pytest.raises(ValueError, match="uint8"):
        st.put([image((20, 20)).astype(np.int16), image((20, 20))])
    with pytest.raises(ValueError, match="uint8"):
        st.put([image((20, 20))[None], image((20, 20))])
    with pytest.raises(ValueError, match=r"\(N, H, W\)"):
        InputStagerCPU((2, 4, 16, 16), max_source_pixels=1000)
    with pytest.raises(ValueError, match="max_source_pixels"):
        InputStagerCPU((2, 16, 16), max_source_pixels=0)


def test_stager_without_max_source_pixels_is_unchanged(emu):
    st = InputStagerCPU((2, 16, 16))
    assert st.max_source_pixels is None and st.h2d_bytes_per_batch == 2 * 2 * 16 * 16
    batch = np.stack([image((16, 16), 1), image((16, 16), 2)])
    st.put(batch, batch)
    x, y = st.get()
    assert torch.equal(x, OS.zscore_u8(batch)) and emu.resize_calls == []
    with pytest.raises(ValueError, match="shape"):
        st.put(np.stack([image((16, 8)), image((16, 8))]))
