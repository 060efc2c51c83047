#!/usr/bin/env python
"""tests/golden/augment3d.npz: what the reference's 3-D augmenter returns.

Build container only (needs a reference checkout named by $PYTORCHDEEPLEARING_REFERENCE; the augmenter imports only
numpy and scipy, ``ImageAugmentation`` also pandas, so the unmodified modules are imported without stubs):
    PYTORCHDEEPLEARING_REFERENCE=/path/to/PytorchDeepLearing python tests/golden/make_golden_augment3d.py

For every case (``<case>_*``): the inputs, the seed, the generator's options (``cfg``, JSON; ``rescale_kind`` says
whether ``rescale`` was a Python float or a numpy float64), every value numpy's global RNG returned to the augmenter in
order (``draws``: ``np.random.uniform`` / ``np.random.random`` are wrapped by recorders while the reference runs), the
centred 4x4 matrix of every sample (recorded from the module's ``apply_transform``), the outputs, and the RNG state
after the call (``state_keys``, ``state_pos``).  Cases:
  - ``rt_*``: ``random_transform(x, y)`` -- every fill mode ('constant' with cval 2.5), ``Augmain.py``'s options on an
    anisotropic (16, 40, 48) volume, a channel shift with C = 3, C = 4, ``depth_flip`` with a unit axis, uint8 labels
    under 'constant' with cval 3.7;
  - ``flow_*``: ``flow(X, y, batch_size, shuffle=True, seed)`` for several batches including a short last one, under
    ``DataAug3D``'s defaults (rescale 1.1 as a Python float), ``rescale=np.float64(1.1)``, ``rescale=None`` and a channel
    shift with C = 3 (``bsizes`` the batch sizes, outputs concatenated);
  - ``da3d_*``: ``DataAug3D(Augmain.py's options).DataAugmentation(csv, number=3, aug_path)`` on two tiny ``.npy``
    pairs listed in a temporary CSV: the inputs and every written file (``img_<index>_<i>``, ``mask_<index>_<i>``).
Inputs hold distinct values, so a wrong source index changes bits."""
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYTORCHDEEPLEARING_REFERENCE")
if not REF:
    sys.exit("set PYTORCHDEEPLEARING_REFERENCE to the reference checkout")
sys.path.insert(0, REF)
from dataprocess.Augmentation import images_masks_3dtransform as T  # noqa: E402
from dataprocess.Augmentation import ImageAugmentation as IA  # noqa: E402


class Recorder:
    """records numpy's draws and the matrices while the reference runs"""

    def __init__(self):
        self.draws, self.matrices = [], []

    def __enter__(self):
        self._u, self._r, self._a = np.random.uniform, np.random.random, T.apply_transform
        rec = self

        def uniform(*a, **k):
            v = rec._u(*a, **k)
            rec.draws.extend(np.atleast_1d(np.asarray(v, dtype=np.float64)).tolist())
            return v

        def random(*a, **k):
            v = rec._r(*a, **k)
            rec.draws.extend(np.atleast_1d(np.asarray(v, dtype=np.float64)).tolist())
            return v

        def apply_transform(x, transform_matrix, *a, **k):
            rec.matrices.append(np.array(transform_matrix, dtype=np.float64))
            return rec._a(x, transform_matrix, *a, **k)

        np.random.uniform, np.random.random, T.apply_transform = uniform, random, apply_transform
        return self

    def __exit__(self, *exc):
        np.random.uniform, np.random.random, T.apply_transform = self._u, self._r, self._a

    def sample_matrices(self):
        return np.stack(self.matrices[0::2])      # apply_transform runs for x, then for y, per sample


def distinct(rng, shape, dtype=np.float32):
    n = int(np.prod(shape))
    return (rng.permutation(n).astype(np.float64) * 0.37 + 1.25).astype(dtype).reshape(shape)


def record_state(out, key):
    st = np.random.get_state()
    out[key + "_state_keys"] = st[1].copy()
    out[key + "_state_pos"] = np.int64(st[2])


def cfg_of(kw):
    c = dict(kw)
    r = c.get("rescale")
    c["rescale_kind"] = None if r is None else ("float64" if isinstance(r, np.float64) else "float")
    if r is not None:
        c["rescale"] = float(r)
    return json.dumps(c)


RT_CASES = {
    # name: (generator options, (D, H, W, C), label dtype, seed)
    "rt_augmain": (dict(rotation_range=10, width_shift_range=0.01, height_shift_range=0.01, depth_shift_range=0,
                        zoom_range=0, horizontal_flip=True, vertical_flip=True, rescale=1.1, fill_mode="nearest"),
                   (16, 40, 48, 1), np.float32, 11),
    "rt_nearest": (dict(rotation_range=25, width_shift_range=0.1, height_shift_range=0.1, depth_shift_range=0.1,
                        zoom_range=0.2, fill_mode="nearest"), (9, 10, 7, 1), np.float32, 1),
    "rt_constant": (dict(rotation_range=25, width_shift_range=0.1, height_shift_range=0.1, depth_shift_range=0.1,
                         zoom_range=0.2, fill_mode="constant", cval=2.5), (9, 10, 7, 1), np.float32, 2),
    "rt_reflect": (dict(rotation_range=25, width_shift_range=0.2, height_shift_range=0.2, depth_shift_range=0.2,
                        zoom_range=0.3, fill_mode="reflect"), (9, 10, 7, 1), np.float32, 3),
    "rt_wrap": (dict(rotation_range=25, width_shift_range=0.2, height_shift_range=0.2, depth_shift_range=0.2,
                     zoom_range=0.3, fill_mode="wrap"), (9, 10, 7, 1), np.float32, 4),
    "rt_mirror": (dict(rotation_range=25, width_shift_range=0.2, height_shift_range=0.2, depth_shift_range=0.2,
                       zoom_range=0.3, fill_mode="mirror"), (9, 10, 7, 1), np.float32, 5),
    "rt_shift_c3": (dict(rotation_range=15, zoom_range=0.1, channel_shift_range=40.0, fill_mode="nearest"),
                    (8, 9, 11, 3), np.float32, 6),
    "rt_c4": (dict(rotation_range=30, height_shift_range=0.1, zoom_range=[0.8, 1.1], vertical_flip=True),
              (6, 7, 8, 4), np.float32, 7),
    "rt_depthflip_unit": (dict(rotation_range=8, depth_flip=True, horizontal_flip=True, zoom_range=0.05),
                          (10, 8, 1, 1), np.float32, 8),
    "rt_u8_constant": (dict(rotation_range=20, width_shift_range=0.15, fill_mode="constant", cval=3.7),
                       (7, 8, 9, 1), np.uint8, 9),
}

FLOW_CASES = {
    # name: (generator options, (N, D, H, W, C), batch_size, seed, batches)
    "flow_defaults": (dict(rotation_range=5, width_shift_range=0.01, height_shift_range=0.01, depth_shift_range=0.01,
                           zoom_range=0.01, rescale=1.1, horizontal_flip=True, vertical_flip=False, depth_flip=False,
                           fill_mode="nearest"), (3, 8, 10, 12, 1), 2, 7, 4),
    "flow_rescale64": (dict(rotation_range=12, zoom_range=0.1, rescale=np.float64(1.1), vertical_flip=True),
                       (2, 9, 8, 7, 1), 2, 3, 2),
    "flow_rescale_none": (dict(rotation_range=12, zoom_range=0.1, rescale=None, depth_flip=True),
                          (2, 9, 8, 7, 1), 2, 5, 2),
    "flow_shift_c3": (dict(rotation_range=12, channel_shift_range=30.0, rescale=1.1, horizontal_flip=True),
                      (3, 6, 7, 8, 3), 2, 9, 2),
}


def main():
    out = {}
    rng = np.random.RandomState(2026)
    for name, (kw, shape, ydt, seed) in RT_CASES.items():
        gen = T.ImageDataGenerator3D(**kw)
        x = distinct(rng, shape)
        y = distinct(rng, shape[:3] + (1,)) if ydt == np.float32 else \
            rng.randint(0, 256, shape[:3] + (1,)).astype(np.uint8)
        np.random.seed(seed)
        with Recorder() as rec:
            xo, yo = gen.random_transform(x.copy(), y.copy())
        out.update({f"{name}_x": x, f"{name}_y": y, f"{name}_seed": np.int64(seed), f"{name}_cfg": cfg_of(kw),
                    f"{name}_draws": np.array(rec.draws), f"{name}_matrices": rec.sample_matrices(),
                    f"{name}_xo": np.ascontiguousarray(xo), f"{name}_yo": np.ascontiguousarray(yo)})
        record_state(out, name)
    for name, (kw, shape, bs, seed, nb) in FLOW_CASES.items():
        gen = T.ImageDataGenerator3D(**kw)
        X = distinct(rng, shape)
        Y = distinct(rng, shape[:4] + (1,))
        it = gen.flow(X, Y, batch_size=bs, shuffle=True, seed=seed)
        bx, by, sizes = [], [], []
        with Recorder() as rec:
            for _ in range(nb):
                a, b = next(it)
                bx.append(a)
                by.append(b)
                sizes.append(a.shape[0])
        out.update({f"{name}_x": X, f"{name}_y": Y, f"{name}_seed": np.int64(seed), f"{name}_cfg": cfg_of(kw),
                    f"{name}_batch_size": np.int64(bs), f"{name}_bsizes": np.array(sizes),
                    f"{name}_draws": np.array(rec.draws), f"{name}_matrices": rec.sample_matrices(),
                    f"{name}_xo": np.concatenate(bx), f"{name}_yo": np.concatenate(by)})
        record_state(out, name)
    # DataAug3D.DataAugmentation itself, with Augmain.py's options
    kw = dict(rotation=10, width_shift=0.01, height_shift=0.01, depth_shift=0, zoom_range=0, vertical_flip=True,
              horizontal_flip=True)
    number, seed = 3, 21
    with tempfile.TemporaryDirectory() as tmp:
        rows = []
        for i, shape in enumerate(((8, 12, 10), (6, 9, 11))):
            img = distinct(rng, shape)
            mask = rng.randint(0, 256, shape).astype(np.uint8)
            np.save(os.path.join(tmp, f"img{i}.npy"), img)
            np.save(os.path.join(tmp, f"mask{i}.npy"), mask)
            out[f"da3d_src_img_{i}"], out[f"da3d_src_mask_{i}"] = img, mask
            rows.append(f"{os.path.join(tmp, f'img{i}.npy')},{os.path.join(tmp, f'mask{i}.npy')}")
        csv = os.path.join(tmp, "train.csv")
        with open(csv, "w") as f:
            f.write("Image,Mask\n" + "\n".join(rows) + "\n")
        aug = os.path.join(tmp, "aug") + "/"
        os.makedirs(aug + "Image")
        os.makedirs(aug + "Mask")
        np.random.seed(seed)
        with Recorder() as rec:
            IA.DataAug3D(**kw).DataAugmentation(csv, number, aug_path=aug)
        record_state(out, "da3d")
        for i in range(2):
            for k in range(1, number + 1):
                out[f"da3d_img_{i}_{k}"] = np.load(aug + f"Image/{i}_{k}.npy")
                out[f"da3d_mask_{i}_{k}"] = np.load(aug + f"Mask/{i}_{k}.npy")
        out.update({"da3d_seed": np.int64(seed), "da3d_number": np.int64(number), "da3d_cfg": json.dumps(kw),
                    "da3d_draws": np.array(rec.draws), "da3d_matrices": rec.sample_matrices()})
    path = os.path.join(HERE, "augment3d.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
