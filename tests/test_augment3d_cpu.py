"""CPU tests of the 3-D augmentation (``ImageDataGenerator3D``, pytorchdeeplearing_b200/augment.py): the fp64 oracle
against scipy itself, the oracle against the reference's recorded outputs (tests/golden/augment3d.npz), the host
draws and matrices against the recorded ones, and the Python layer end to end on an emulated backend that runs the
oracle in place of csrc/augment3d.cu.  The reference is not imported."""
import json
import os
import struct
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import augment3d as oa  # noqa: E402
from pytorchdeeplearing_b200 import augment as A, runtime  # noqa: E402
from pytorchdeeplearing_b200._abi import AUG3D_PARAM_BYTES, AUG_MODES, RESCALE_F32, RESCALE_F64  # noqa: E402

ndi = pytest.importorskip("scipy.ndimage")
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "augment3d.npz"))
RT_CASES = sorted({k[:-4] for k in GOLD.files if k.startswith("rt_") and k.endswith("_cfg")})
FLOW_CASES = sorted({k[:-4] for k in GOLD.files if k.startswith("flow_") and k.endswith("_cfg")})
MODE_NAMES = {v: k for k, v in AUG_MODES.items()}


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def gen_kwargs(case):
    cfg = json.loads(str(GOLD[f"{case}_cfg"]))
    kind = cfg.pop("rescale_kind", None)
    if kind == "float64":
        cfg["rescale"] = np.float64(cfg["rescale"])
    return cfg


class DrawRecorder:
    """the values numpy's global RNG hands out through uniform / random while active"""

    def __enter__(self):
        self.draws = []
        self._u, self._r = np.random.uniform, np.random.random
        rec = self

        def uniform(*a, **k):
            v = rec._u(*a, **k)
            rec.draws.extend(np.atleast_1d(np.asarray(v, dtype=np.float64)).tolist())
            return v

        def random(*a, **k):
            v = rec._r(*a, **k)
            rec.draws.extend(np.atleast_1d(np.asarray(v, dtype=np.float64)).tolist())
            return v

        np.random.uniform, np.random.random = uniform, random
        return self

    def __exit__(self, *exc):
        np.random.uniform, np.random.random = self._u, self._r


def rng_state_is(case):
    st = np.random.get_state()
    return np.array_equal(st[1], GOLD[f"{case}_state_keys"]) and st[2] == int(GOLD[f"{case}_state_pos"])


def ulp_close(a, b, n=2):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return bool(np.all(np.abs(a - b) <= n * np.spacing(np.maximum(np.abs(a), np.abs(b)))))


# ------------------------------------------------------------------------------------------- oracle vs scipy
def _check_scipy(v, m, off, mode, cval):
    ref = ndi.affine_transform(v, m, off, order=0, mode=mode, cval=cval)
    got = oa.affine_order0(v, m, off, mode, cval)
    assert bits_equal(ref, got), (mode, m, off, v.shape)


@pytest.mark.parametrize("mode", oa.MODES)
def test_oracle_offset_sweep_matches_scipy(mode):
    """offsets across [-2 len, 2 len] in steps of 0.5 and their +-1 ulp neighbours, per axis length 1..8"""
    for n in (1, 2, 3, 4, 5, 8):
        v = (np.arange(n * 3 * 2, dtype=np.float32) + 1).reshape(n, 3, 2)
        for base in np.arange(-2 * n, 2 * n + 0.5, 0.5):
            for o in (np.nextafter(base, -np.inf), base, np.nextafter(base, np.inf)):
                for s in (1.0, -1.0, 0.5, 2.0):
                    _check_scipy(v, np.diag([s, 1.0, 1.0]), np.array([o, 0.0, 0.0]), mode, 7.5)


@pytest.mark.parametrize("mode", oa.MODES)
def test_oracle_tie_heavy_and_rotations_match_scipy(mode):
    rng = np.random.default_rng(17)
    for _ in range(150):                           # matrix entries and offsets that put coordinates on .5 ties
        shape = tuple(int(s) for s in rng.integers(1, 7, 3))
        v = (np.arange(np.prod(shape), dtype=np.float32) + 1).reshape(shape)
        m = rng.choice([0.1, 0.2, 0.3, 0.6, 0.7, -0.3, 1.0, -1.1, 1.5], (3, 3))
        _check_scipy(v, m, rng.integers(-8, 8, 3) + 0.5, mode, -3.0)
    for shape in ((1, 5, 6), (7, 1, 4), (6, 8, 1), (9, 10, 7), (8, 8, 8), (5, 12, 3)):   # odd, even, unit axes
        v = (np.arange(np.prod(shape), dtype=np.float32) + 1).reshape(shape)
        for _ in range(8):
            a = rng.uniform(-0.35, 0.35, 3)
            cx, sx, cy, sy, cz, sz = np.cos(a[0]), np.sin(a[0]), np.cos(a[1]), np.sin(a[1]), np.cos(a[2]), np.sin(a[2])
            r = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) \
                @ np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
            _check_scipy(v, r * rng.uniform(0.8, 1.2), rng.uniform(-3, 3, 3), mode, 0.0)


@pytest.mark.parametrize("cval", [0.4, 2.5, 3.7, 254.6, 300.0, -3.0])
def test_oracle_uint8_fill_matches_scipy(cval):
    rng = np.random.default_rng(5)
    for _ in range(10):
        shape = tuple(int(s) for s in rng.integers(1, 9, 3))
        v = rng.integers(0, 256, shape).astype(np.uint8)
        _check_scipy(v, np.eye(3) + rng.uniform(-0.4, 0.4, (3, 3)), rng.uniform(-4, 4, 3), "constant", cval)


# ------------------------------------------------------------------------------------------- oracle vs fixtures
def _oracle_on_fixture(case, entries, kw, rescale):
    x, y = GOLD[f"{case}_x"], GOLD[f"{case}_y"]
    if x.ndim == 4:
        x, y = x[None], y[None]
    return oa.warp_batch(x, y[..., 0], entries, kw.get("fill_mode", "nearest"), kw.get("cval", 0.0),
                         kw.get("channel_shift_range", 0) != 0, rescale)


def _recorded_entries(case, kw, shape, channels, count):
    """entries from the RECORDED matrices, with the shifts and flips of the drop-in's own draws (pinned separately)"""
    np.random.seed(int(GOLD[f"{case}_seed"]))
    gen = A.ImageDataGenerator3D(**kw)
    out = []
    for m4 in GOLD[f"{case}_matrices"][:count]:
        d = A.draw_transform(gen, shape, channels)
        shifts = [float(np.float32(u)) for u in d["channel_shift"]] if d["channel_shift"] is not None else []
        out.append((m4[:3, :3].reshape(-1), m4[:3, 3], shifts, A.flip_bits(d["flips"])))
    return out


@pytest.mark.parametrize("case", RT_CASES)
def test_oracle_chain_reproduces_random_transform_fixture(case):
    kw = gen_kwargs(case)
    x = GOLD[f"{case}_x"]
    entries = _recorded_entries(case, kw, x.shape[:3], x.shape[3], 1)
    xo, yo = _oracle_on_fixture(case, entries, kw, None)
    assert bits_equal(xo[0], GOLD[f"{case}_xo"])
    assert bits_equal(yo[0][..., None], GOLD[f"{case}_yo"])


@pytest.mark.parametrize("case", FLOW_CASES)
def test_oracle_chain_reproduces_flow_fixture(case):
    """per batch: the seeded index walk, then the recorded matrices; float64 outputs as NumpyArrayIterator"""
    kw = gen_kwargs(case)
    X, Y = GOLD[f"{case}_x"], GOLD[f"{case}_y"]
    bs, seed = int(GOLD[f"{case}_batch_size"]), int(GOLD[f"{case}_seed"])
    gen = A.ImageDataGenerator3D(**kw)
    it = A.NumpyArrayIterator(X, Y, gen, batch_size=bs, shuffle=True, seed=seed)
    mats = GOLD[f"{case}_matrices"]
    done, xs, ys = 0, [], []
    for size in GOLD[f"{case}_bsizes"]:
        idx, _, cur = next(it.index_generator)
        assert cur == size
        entries = []
        for j in range(cur):
            d = A.draw_transform(gen, X.shape[1:4], X.shape[4])
            shifts = [float(np.float32(u)) for u in d["channel_shift"]] if d["channel_shift"] is not None else []
            m4 = mats[done + j]
            entries.append((m4[:3, :3].reshape(-1), m4[:3, 3], shifts, A.flip_bits(d["flips"])))
        done += cur
        xo, yo = oa.warp_batch(X[idx], Y[idx][..., 0].astype(np.float32), entries, kw.get("fill_mode", "nearest"),
                               kw.get("cval", 0.0), kw.get("channel_shift_range", 0) != 0, kw.get("rescale"))
        xs.append(xo.astype(np.float64))
        ys.append(yo[..., None].astype(np.float64))
    assert bits_equal(np.concatenate(xs), GOLD[f"{case}_xo"])
    assert bits_equal(np.concatenate(ys), GOLD[f"{case}_yo"])
    assert rng_state_is(case)


# ------------------------------------------------------------------------------------------- host draws, matrices
@pytest.mark.parametrize("case", RT_CASES)
def test_host_draws_and_matrices_match_fixture(case):
    kw = gen_kwargs(case)
    x = GOLD[f"{case}_x"]
    gen = A.ImageDataGenerator3D(**kw)
    np.random.seed(int(GOLD[f"{case}_seed"]))
    with DrawRecorder() as rec:
        d = A.draw_transform(gen, x.shape[:3], x.shape[3])
    assert np.array_equal(np.array(rec.draws), GOLD[f"{case}_draws"])
    assert rng_state_is(case)
    m = A.compose_matrix(d, x.shape[:3])
    # the same np.dot chain, evaluated here
    th = d["theta"]
    c, s = np.cos, np.sin
    rx = np.array([[1, 0, 0, 0], [0, c(th[0]), -s(th[0]), 0], [0, s(th[0]), c(th[0]), 0], [0, 0, 0, 1]])
    ry = np.array([[c(th[1]), 0, s(th[1]), 0], [0, 1, 0, 0], [-s(th[1]), 0, c(th[1]), 0], [0, 0, 0, 1]])
    rz = np.array([[c(th[2]), -s(th[2]), 0, 0], [s(th[2]), c(th[2]), 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    t = np.array([[1, 0, 0, d["shift"][0]], [0, 1, 0, d["shift"][1]], [0, 0, 1, d["shift"][2]], [0, 0, 0, 1]])
    z = np.array([[d["zoom"][0], 0, 0, 0], [0, d["zoom"][1], 0, 0], [0, 0, d["zoom"][2], 0], [0, 0, 0, 1]])
    o = [float(n) / 2 + 0.5 for n in x.shape[:3]]
    om = np.array([[1, 0, 0, o[0]], [0, 1, 0, o[1]], [0, 0, 1, o[2]], [0, 0, 0, 1]])
    rm = np.array([[1, 0, 0, -o[0]], [0, 1, 0, -o[1]], [0, 0, 1, -o[2]], [0, 0, 0, 1]])
    want = np.dot(np.dot(om, np.dot(np.dot(np.dot(np.dot(rx, ry), rz), t), z)), rm)
    assert bits_equal(m, want)
    assert ulp_close(m, GOLD[f"{case}_matrices"][0])


def test_host_draw_order_and_types():
    gen = A.ImageDataGenerator3D(rotation_range=10, width_shift_range=0.1, height_shift_range=0.2,
                                 depth_shift_range=0.3, zoom_range=0.1, channel_shift_range=2.0,
                                 horizontal_flip=True, vertical_flip=True, depth_flip=True)
    np.random.seed(0)
    d = A.draw_transform(gen, (10, 20, 30), 3)
    np.random.seed(0)
    u = [np.random.uniform(-10, 10) for _ in range(3)]
    sh = [np.random.uniform(-0.2, 0.2) * 10, np.random.uniform(-0.1, 0.1) * 20, np.random.uniform(-0.3, 0.3) * 30]
    z = np.random.uniform(0.9, 1.1, 3)
    cs = [np.random.uniform(-2.0, 2.0) for _ in range(3)]
    f = [np.random.random() < 0.5 for _ in range(3)]      # horizontal (axis 1), vertical (axis 0), depth (axis 2)
    assert d["theta"] == tuple(np.pi / 180 * v for v in u) and d["shift"] == tuple(sh)
    assert d["zoom"] == tuple(z) and d["channel_shift"] == cs and d["flips"] == (f[1], f[0], f[2])
    assert A.ImageDataGenerator3D().zoom_range == [1, 1]
    assert A.ImageDataGenerator3D(zoom_range=0.2).zoom_range == [0.8, 1.2]
    assert A.ImageDataGenerator3D(zoom_range=(0.5, 2)).zoom_range == [0.5, 2]


def test_rescale_forms():
    assert A.rescale_form(None)[0] == 0 and A.rescale_form(0)[0] == 0
    assert A.rescale_form(1.1) == (RESCALE_F32, 1.1)
    assert A.rescale_form(2)[0] == RESCALE_F32 and A.rescale_form(np.float32(1.1))[0] == RESCALE_F32
    assert A.rescale_form(np.float64(1.1)) == (RESCALE_F64, 1.1)
    x = np.random.default_rng(0).standard_normal(10000).astype(np.float32)
    for r in (1.1, np.float64(1.1), 3, np.float32(0.7)):
        want = x.copy()
        want *= r
        assert bits_equal(oa.rescale_sample(x, r), want)


def test_unsupported_options_raise():
    for kw in (dict(featurewise_center=True), dict(featurewise_std_normalization=True), dict(zca_whitening=True),
               dict(samplewise_center=True), dict(samplewise_std_normalization=True), dict(dim_ordering="th"),
               dict(fill_mode="grid-wrap")):
        with pytest.raises(NotImplementedError):
            A.ImageDataGenerator3D(**kw)
    with pytest.raises(ValueError):
        A.ImageDataGenerator3D(dim_ordering="xy")
    with pytest.raises(ValueError):
        A.ImageDataGenerator3D(zoom_range=(1, 2, 3))
    g = A.ImageDataGenerator3D(preprocessing_function=abs)
    assert g.preprocessing_function is abs


# ------------------------------------------------------------------------------------------- Python layer, emulated
class EmuAugBackend:
    """``CudaBackend.augment3d`` restated by the oracle on CPU tensors"""

    def __init__(self):
        self.launches = 0

    def augment3d_workspace(self, n, dhw, device):
        return torch.empty(16, dtype=torch.uint8)

    def augment3d(self, x, y, params, x_out, y_out, mode=0, cval=0.0, shift=False, rescale=0.0, rescale_mode=0,
                  binarize=False, ws=None):
        raw = params.numpy().tobytes()
        entries = []
        for s in range(x.shape[0]):
            v = struct.unpack_from("<9d3d4fii", raw, s * AUG3D_PARAM_BYTES)
            entries.append((v[:9], v[9:12], v[12:12 + x.shape[4]], v[16]))
        r = None if rescale_mode == 0 else (rescale if rescale_mode == RESCALE_F32 else np.float64(rescale))
        lo = "binary" if binarize else ("int64" if y_out.dtype == torch.int64 else None)
        xo, yo = oa.warp_batch(x.numpy(), y.numpy(), entries, MODE_NAMES[mode], cval, shift, r, lo)
        x_out.copy_(torch.from_numpy(xo))
        y_out.copy_(torch.from_numpy(yo))
        self.launches += 1


@pytest.fixture
def emu():
    if torch.cuda.is_available():
        pytest.skip("the emulated backend runs on CPU tensors")
    be = EmuAugBackend()
    runtime._set_backend_for_testing(be)
    yield be
    runtime._set_backend_for_testing(None)


@pytest.mark.parametrize("case", RT_CASES)
def test_random_transform_python_layer(emu, case):
    kw = gen_kwargs(case)
    gen = A.ImageDataGenerator3D(**kw)
    np.random.seed(int(GOLD[f"{case}_seed"]))
    xo, yo = gen.random_transform(GOLD[f"{case}_x"], GOLD[f"{case}_y"])
    assert rng_state_is(case) and emu.launches == 1
    x = GOLD[f"{case}_x"]
    np.random.seed(int(GOLD[f"{case}_seed"]))
    m = A.compose_matrix(A.draw_transform(gen, x.shape[:3], x.shape[3]), x.shape[:3])
    if bits_equal(m, GOLD[f"{case}_matrices"][0]):
        assert bits_equal(xo, GOLD[f"{case}_xo"]) and bits_equal(yo, GOLD[f"{case}_yo"])
    else:      # a BLAS / libm that differs from the recording's in the last bit: the oracle on our own matrices
        entries = _recorded_entries(case, kw, x.shape[:3], x.shape[3], 1)
        entries[0] = (m[:3, :3].reshape(-1), m[:3, 3]) + entries[0][2:]
        wx, wy = _oracle_on_fixture(case, entries, kw, None)
        assert bits_equal(xo, wx[0]) and bits_equal(yo, wy[0][..., None])


@pytest.mark.parametrize("case", FLOW_CASES)
def test_flow_python_layer(emu, case):
    kw = gen_kwargs(case)
    gen = A.ImageDataGenerator3D(**kw)
    it = gen.flow(GOLD[f"{case}_x"], GOLD[f"{case}_y"], batch_size=int(GOLD[f"{case}_batch_size"]),
                  seed=int(GOLD[f"{case}_seed"]))
    xs, ys = zip(*[next(it) for _ in GOLD[f"{case}_bsizes"]])
    assert emu.launches == len(GOLD[f"{case}_bsizes"]) and rng_state_is(case)
    assert xs[0].dtype == np.float64 and ys[0].dtype == np.float64
    assert [a.shape[0] for a in xs] == list(GOLD[f"{case}_bsizes"])
    # on a machine whose BLAS reproduces the recorded matrices this is the fixture itself
    np.random.seed(int(GOLD[f"{case}_seed"]))
    X = GOLD[f"{case}_x"]
    same = True
    it2 = A.NumpyArrayIterator(X, GOLD[f"{case}_y"], gen, batch_size=int(GOLD[f"{case}_batch_size"]), shuffle=True,
                               seed=int(GOLD[f"{case}_seed"]))
    k = 0
    for size in GOLD[f"{case}_bsizes"]:
        next(it2.index_generator)
        for _ in range(size):
            m = A.compose_matrix(A.draw_transform(gen, X.shape[1:4], X.shape[4]), X.shape[1:4])
            same &= bits_equal(m, GOLD[f"{case}_matrices"][k])
            k += 1
    if same:
        assert bits_equal(np.concatenate(xs), GOLD[f"{case}_xo"]) and bits_equal(np.concatenate(ys), GOLD[f"{case}_yo"])


def test_transform_batch_python_layer(emu):
    rng = np.random.default_rng(3)
    x = torch.from_numpy(rng.standard_normal((3, 1, 6, 7, 8)).astype(np.float32))
    y = torch.from_numpy(rng.integers(0, 3, (3, 6, 7, 8)).astype(np.uint8))
    gen = A.ImageDataGenerator3D(rotation_range=10, zoom_range=0.1, horizontal_flip=True, rescale=1.1)
    np.random.seed(4)
    xo, yo = gen.transform_batch(x, y)
    assert emu.launches == 1 and xo.shape == x.shape and yo.dtype == torch.int64
    np.random.seed(4)
    for s in range(3):
        xs, ys = gen.random_transform(x[s, 0, ..., None].numpy(), y[s, ..., None].numpy())
        assert bits_equal(xo[s, 0].numpy(), oa.rescale_sample(xs, 1.1)[..., 0])
        assert bits_equal(yo[s].numpy(), (ys[..., 0] != 0).astype(np.int64))


# ------------------------------------------------------------------------------------------- install()
def test_install_rebinds_the_augmentation_modules(monkeypatch):
    import pytorchdeeplearing_b200 as b200
    names = ("dataprocess.Augmentation.images_masks_3dtransform", "dataprocess.Augmentation.ImageAugmentation")

    class Original:
        pass

    mods = []
    for name in names:
        m = types.ModuleType(name)
        m.ImageDataGenerator3D = Original
        monkeypatch.setitem(sys.modules, name, m)
        mods.append(m)
    try:
        assert b200.install() >= 2
        assert all(m.ImageDataGenerator3D is b200.ImageDataGenerator3D for m in mods)
    finally:
        b200.uninstall()
    assert all(m.ImageDataGenerator3D is Original for m in mods)
