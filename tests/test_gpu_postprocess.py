"""Mask post-processing on the GPU (b200seg_largest_component / b200seg_morphology / b200seg_label_bbox,
csrc/postprocess.cu): exact equality with the scipy oracle (oracle/postprocess.py) on random masks, adversarial
component layouts, odd shapes, a CT-sized volume, every radius class and predict_mask output; guard bands around
outputs, bit-identical reruns and CUDA-graph replay on new mask contents."""
import numpy as np
import pytest
import torch
from scipy import ndimage

from oracle import postprocess as opp
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import runtime

pytestmark = pytest.mark.gpu
GUARD = 64          # guard bytes before and after every output
OPS = opp.OPS


def dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def check_cc(m, t=None):
    out, st = b200.largest_component(dev(m) if t is None else t)
    want, n, big = opp.largest_component(m)
    assert st.tolist() == [n, big]
    assert out.dtype == torch.uint8 and out.shape == m.shape
    assert np.array_equal(out.cpu().numpy(), want)


def check_bbox(m, t=None):
    box = b200.label_bbox(dev(m) if t is None else t)
    assert box.tolist() == opp.label_bbox(m).tolist()


def check_morph(m, r, op, want=None, t=None):
    out = b200.binary_morphology(dev(m) if t is None else t, r, op)
    want = opp.morphology(m, r, op) if want is None else want
    got = out.cpu().numpy()
    assert out.dtype == torch.uint8 and got.shape == m.shape
    if not np.array_equal(got, want):
        bad = np.argwhere(got != want)
        raise AssertionError(f"{op} r={r} shape {m.shape}: {len(bad)} voxels differ, first {bad[0].tolist()} "
                             f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}")


def blobs(shape, density, seed, sigma=1.5):
    """smooth random blobs with about ``density`` foreground"""
    f = ndimage.gaussian_filter(np.random.default_rng(seed).random(shape), sigma)
    return (f > np.quantile(f, 1 - density)).astype(np.uint8)


# exact squared-distance restatement for radii where scipy's per-offset ball loop is too slow: scipy's exact EDT
# gives a nearest seed's index, so the squared distance is an integer
def edt_dilate(fg, r):
    if not fg.any():
        return np.zeros(fg.shape, bool)
    idx = ndimage.distance_transform_edt(~fg, return_distances=False, return_indices=True)
    grid = np.indices(fg.shape)
    d2 = sum((idx[a].astype(np.int64) - grid[a]) ** 2 for a in range(fg.ndim))
    return d2 <= r * r + r


def edt_morph(m, r, op):
    fg = m != 0

    def ero(x):
        return ~edt_dilate(~x, r)

    if op == "dilate":
        out = edt_dilate(fg, r)
    elif op == "erode":
        out = ero(fg)
    elif op == "open":
        out = edt_dilate(ero(fg), r)
    else:
        out = ero(edt_dilate(np.pad(fg, r), r))[tuple(slice(r, r + s) for s in fg.shape)]
    return out.astype(np.uint8)


# ------------------------------------------------------------------------------------------------ random masks
MASK_DTYPES = [torch.bool, torch.uint8, torch.int16, torch.int32, torch.int64]


@pytest.mark.parametrize("density", [0.05, 0.3116, 0.9])
@pytest.mark.parametrize("shape", [(40, 56, 72), (300, 260)])
def test_random_masks(density, shape):
    rng = np.random.default_rng(int(density * 1e4) + len(shape))
    m = (rng.random(shape) < density).astype(np.uint8)
    for dt in MASK_DTYPES:
        check_cc(m, dev(m, dt))
    lab = m * rng.integers(1, 3, shape).astype(np.uint8)         # values 0, 1, 2: the box counts only 1
    for dt in MASK_DTYPES[1:]:
        check_bbox(lab, dev(lab, dt))
    check_bbox(m, dev(m, torch.bool))
    for op in OPS:
        check_morph(m, 1, op)
        check_morph(m, 2, op, t=dev(lab, torch.float32))


def test_morphology_float_mask_counts_nan_as_foreground():
    m = blobs((20, 30, 40), 0.3, 3).astype(np.float32) * 0.25
    m[np.random.default_rng(4).random(m.shape) < 0.01] = np.nan
    m[0, 0, 0] = -0.0
    for op in OPS:
        check_morph(m, 2, op)


# ------------------------------------------------------------------------------------------------ layouts
def serpentine(D, H, W):
    """one path through every tile: full rows on even (z, y), joined at alternating ends, layers joined at a corner"""
    m = np.zeros((D, H, W), np.uint8)
    ys = list(range(0, H, 2))
    for k, z in enumerate(range(0, D, 2)):
        order = ys if k % 2 == 0 else ys[::-1]
        for j, y in enumerate(order):
            m[z, y] = 1
            if j + 1 < len(order):
                m[z, min(y, order[j + 1]) + 1, W - 1 if j % 2 == 0 else 0] = 1
        if z + 2 < D:
            m[z + 1, order[-1], W - 1 if (len(order) - 1) % 2 == 0 else 0] = 1
    return m


def test_serpentine_path_is_one_component():
    m = serpentine(15, 41, 70)
    assert opp.largest_component(m)[1] == 1
    m[1, 1, 35] = 1                                 # a separate single voxel
    assert opp.largest_component(m)[1:] == (2, int(m.sum()) - 1)
    check_cc(m)
    check_cc(serpentine(1, 63, 200)[0])            # the 2-D form
    check_cc(np.ascontiguousarray(serpentine(9, 50, 33).transpose(2, 1, 0)))


def test_checkerboard_every_voxel_its_own_component():
    m = (np.indices((20, 24, 40)).sum(axis=0) % 2).astype(np.uint8)
    out, st = b200.largest_component(dev(m))
    assert st.tolist() == [int(m.sum()), 1]
    first = int(np.flatnonzero(m.ravel())[0])
    assert torch.nonzero(out.flatten()).flatten().tolist() == [first]
    check_cc(m)
    check_cc(1 - m)
    check_cc((np.indices((50, 70)).sum(axis=0) % 2).astype(np.uint8))


def test_equal_sizes_tie_to_the_first_voxel():
    m = np.zeros((16, 40, 40), np.uint8)
    m[10:12, 30:33, 30:33] = 1                      # same size, later
    m[2:4, 20:23, 1:4] = 1                          # same size, first in C order
    m[2:4, 0:3, 35:38] = 1                          # same size, earlier still (smaller y in the same z)
    check_cc(m)
    out, _ = b200.largest_component(dev(m))
    assert out[2, 0, 35].item() == 1 and out.sum().item() == 18


def test_all_foreground_empty_and_objects_on_every_face():
    for shape in ((33, 47, 65), (70, 90)):
        full, empty = np.ones(shape, np.uint8), np.zeros(shape, np.uint8)
        check_cc(full)
        check_cc(empty)
        check_bbox(full)
        check_bbox(empty)
        for op in OPS:
            check_morph(full, 3, op)
            check_morph(empty, 3, op)
    m = np.zeros((33, 47, 65), np.uint8)
    m[0, 5:20, 5:30] = m[-1, 30:40, 10:60] = 1
    m[3:30, 0, 3:9] = m[4:9, -1, :] = 1
    m[:, 20:25, 0] = m[10:20, 10:40, -1] = 1
    m[10:20, 10:40, -3:] = 1
    check_cc(m)
    check_bbox(m)
    for op in OPS:
        for r in (1, 4):
            check_morph(m, r, op)


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 1, 1000), (1000, 1, 1), (37, 41, 43), (1, 5000), (5000, 1), (1, 1)])
def test_odd_shapes(shape):
    rng = np.random.default_rng(sum(shape))
    for m in ((rng.random(shape) < 0.3116).astype(np.uint8), np.ones(shape, np.uint8)):
        check_cc(m)
        check_bbox(m)
        for op in OPS:
            check_morph(m, 2, op)


# ------------------------------------------------------------------------------------------------ CT size
def test_ct_sized_ellipsoid_with_noise_islands():
    sh = (300, 512, 512)
    z, y, x = np.ogrid[:sh[0], :sh[1], :sh[2]]
    m = ((((z - 150) / 110.0) ** 2 + ((y - 250) / 190.0) ** 2 + ((x - 260) / 170.0) ** 2) <= 1).astype(np.uint8)
    rng = np.random.default_rng(7)
    m[rng.random(sh) < 2e-4] = 1
    m[20:40, 20:60, 400:500] = 1                    # a second large object, smaller than the ellipsoid
    t = dev(m)
    check_cc(m, t)
    check_bbox(m, t)
    check_morph(m, 1, "open", t=t)


# ------------------------------------------------------------------------------------------------ radii
@pytest.mark.parametrize("op", OPS)
def test_radii_3d(op):
    m = blobs((18, 30, 34), 0.35, 11)
    for r in (0, 1, 2, 3, 5, 12):
        check_morph(m, r, op)
    small = blobs((5, 40, 44), 0.3, 12, sigma=2.0)
    assert np.array_equal(edt_morph(small, 5, op), opp.morphology(small, 5, op))     # the restatement agrees
    check_morph(small, 64, op, want=edt_morph(small, 64, op))


@pytest.mark.parametrize("op", OPS)
def test_radii_2d(op):
    m = blobs((64, 80), 0.35, 13)
    for r in (0, 1, 2, 3, 5, 12, 64):
        check_morph(m, r, op)


def test_one_slice_3d_close_is_closed_in_3d():
    m = blobs((1, 30, 34), 0.4, 14)
    for r in (1, 3, 5):
        check_morph(m, r, "close")
        check_morph(m[0], r, "close")
    check_morph(m, 64, "close", want=edt_morph(m, 64, "close"))


def test_radius_limits():
    t = dev(np.ones((3, 4, 5), np.uint8))
    with pytest.raises(ValueError, match="radius"):
        b200.binary_morphology(t, 65, "dilate")
    be = runtime.cuda_backend()
    out = torch.empty_like(t)
    with pytest.raises(RuntimeError, match="bad arguments"):
        be.morphology(t, 65, 0, out)


# ------------------------------------------------------------------------------------------------ guard bands
def guarded(n, dtype):
    item = torch.empty((), dtype=dtype).element_size()
    buf = torch.full((GUARD + n * item + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
    return buf, buf[GUARD:GUARD + n * item].view(dtype)


def intact(buf):
    return bool((buf[:GUARD] == 0xA5).all()) and bool((buf[-GUARD:] == 0xA5).all())


@pytest.mark.parametrize("shape", [(37, 41, 43), (61, 77)])
def test_outputs_stay_inside_their_buffers(shape):
    be = runtime.cuda_backend()
    m = blobs(shape, 0.3, 21)
    t = dev(m)
    n = m.size
    ob, out = guarded(n, torch.uint8)
    sb, stats = guarded(2, torch.int64)
    be.largest_component(t, out.view(shape), stats)
    want, nc, big = opp.largest_component(m)
    assert intact(ob) and intact(sb)
    assert np.array_equal(out.view(shape).cpu().numpy(), want) and stats.tolist() == [nc, big]
    for op, code in b200._abi.MORPH_OPS.items():
        ob, out = guarded(n, torch.uint8)
        be.morphology(t, 3, code, out.view(shape))
        assert intact(ob) and np.array_equal(out.view(shape).cpu().numpy(), opp.morphology(m, 3, op))
    bb, box = guarded(2 * len(shape) + 1, torch.int64)
    be.label_bbox(t, box)
    assert intact(bb) and box.tolist() == opp.label_bbox(m).tolist()


# ------------------------------------------------------------------------------------------------ determinism, graphs
def test_reruns_are_bit_identical():
    rng = np.random.default_rng(31)
    t = dev((rng.random((64, 96, 96)) < 0.3116).astype(np.uint8))
    a = [b200.largest_component(t), b200.binary_morphology(t, 3, "close"), b200.label_bbox(t)]
    for _ in range(3):
        b = [b200.largest_component(t), b200.binary_morphology(t, 3, "close"), b200.label_bbox(t)]
        assert torch.equal(a[0][0], b[0][0]) and torch.equal(a[0][1], b[0][1])
        assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


def test_device_forms_replay_in_a_cuda_graph():
    shape = (40, 48, 56)
    masks = [blobs(shape, d, s) for d, s in ((0.3, 41), (0.1, 42), (0.6, 43))]
    static = dev(masks[0])
    b200.largest_component(static)
    b200.binary_morphology(static, 2, "close")
    b200.label_bbox(static)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cc, st = b200.largest_component(static)
        mo = b200.binary_morphology(static, 2, "close")
        box = b200.label_bbox(static)
    for m in masks[1:] + masks[:1]:
        static.copy_(dev(m))
        g.replay()
        torch.cuda.synchronize()
        want, n, big = opp.largest_component(m)
        assert np.array_equal(cc.cpu().numpy(), want) and st.tolist() == [n, big]
        assert np.array_equal(mo.cpu().numpy(), opp.morphology(m, 2, "close"))
        assert box.tolist() == opp.label_bbox(m).tolist()


# ------------------------------------------------------------------------------------------------ wrappers, predict_mask
def test_reference_named_wrappers_on_numpy():
    m = blobs((30, 40, 50), 0.2, 51)
    want = opp.largest_component(m)[0]
    out = b200.GetLargestConnectedCompont(m)
    assert out.dtype == np.uint32 and np.array_equal(out, want)
    assert (b200.GetLargestConnectedCompont(np.zeros((4, 5, 6), np.uint8)) == 1).all()
    for op in OPS:
        assert np.array_equal(b200.MorphologicalOperation(m, 2, op), opp.morphology(m, 2, op))
    assert b200.GetLargestConnectedCompontBoundingbox(m).tolist() == opp.label_bbox(m)[:-1].tolist()
    with pytest.raises(RuntimeError):
        b200.GetLargestConnectedCompontBoundingbox(m * 255)


def test_predict_mask_output_feeds_the_post_processing_directly():
    import oracle
    from oracle import nets as onets
    prev = runtime.get_precision()
    b200.set_precision("bf16")
    try:
        sd = onets.init_state_dict(onets.vnet3d_state_spec(1, 2), seed=0, randomize_affine=True)
        model = b200.VNet3d(1, 2)
        model.load_state_dict(sd)
        model = model.cuda().eval()
        x, _ = oracle.make_inputs(2, 1, (32, 32, 32), 2)
        mask = b200.predict_mask(model, x.cuda())               # uint8 (2, 32, 32, 32) on the device, 0/1
    finally:
        b200.set_precision(prev)
    assert mask.dtype == torch.uint8 and mask.is_cuda
    for n in range(2):
        t = mask[n]
        mh = t.cpu().numpy()
        check_cc(mh, t)
        check_bbox(mh, t)
        for op in OPS:
            check_morph(mh, 1, op, t=t)
