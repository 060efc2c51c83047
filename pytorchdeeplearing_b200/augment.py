"""The reference's 3-D data augmentation on the GPU: ``ImageDataGenerator3D`` (dataprocess/Augmentation/
images_masks_3dtransform.py), as ``DataAug3D`` (dataprocess/Augmentation/ImageAugmentation.py:26-75) drives it to
write augmented ``.npy`` copies of the 3-D training volumes.

Every random draw and the 4x4 matrix stay on the host, with numpy's global legacy RNG and the same numpy calls as the
reference, so a seed gives the reference's parameters and leaves the RNG in the reference's state.  The warp itself --
``scipy.ndimage.affine_transform(order=0)`` of each image channel and of the label, the channel shift, the flips and
``standardize``'s ``x *= rescale`` -- is one launch of ``csrc/augment3d.cu`` for a whole batch, bit for bit scipy's.

    gen = ImageDataGenerator3D(rotation_range=10, horizontal_flip=True, vertical_flip=True, rescale=1.1)
    x2, y2 = gen.random_transform(x, y)            # numpy (D, H, W, C) fp32, (D, H, W, 1) -> the reference's arrays
    for bx, by in gen.flow(X, Y, batch_size=1):    # float64 batches, as NumpyArrayIterator
        ...
    xs, ys = gen.transform_batch(x_dev, y_dev)     # per training step: (N, 1, D, H, W) fp32 + (N, D, H, W) uint8 on
                                                   # the device -> fp32 images, int64 labels (y != 0)

Differences from the reference, all for options it cannot run or ``DataAug3D`` never sets: ``featurewise_*``,
``zca_whitening`` (the reference has no ``fit``, so they fail on ``None``), ``samplewise_*`` and ``dim_ordering='th'``
(the reference leaves its axes unset) raise ``NotImplementedError`` at construction, as does a ``fill_mode`` other
than 'nearest', 'constant', 'reflect', 'wrap' or 'mirror'.  The drop-in takes fp32 images (``flow`` converts, as the
reference does), uint8 or fp32 labels with one channel and the image's spatial shape, and a ``rescale`` that numpy
multiplies in fp32 (a Python number) or fp64 (a numpy float64).  ``preprocessing_function`` is stored and ignored, as
in the reference.
"""
from __future__ import annotations

import threading

import numpy as np
import torch

from . import runtime
from ._abi import AUG_MODES, RESCALE_F32, RESCALE_F64, RESCALE_NONE, aug3d_param_table


# ---------------------------------------------------------------------------------------------- host-only functions
def draw_transform(gen, shape, channels):
    """One sample's draws from numpy's global RNG, in the reference's order (``random_transform``): rotations,
    shifts, zoom, the per-channel shifts (drawn after the warp in the reference, with no draw in between) and the
    flips.  ``shape`` is the sample's (D, H, W).  Returns a dict of the drawn values, in the reference's types."""
    if gen.rotation_range:
        theta = tuple(np.pi / 180 * np.random.uniform(-gen.rotation_range, gen.rotation_range) for _ in range(3))
    else:
        theta = (0, 0, 0)
    shifts = []
    for rng, n in zip((gen.height_shift_range, gen.width_shift_range, gen.depth_shift_range), shape):
        shifts.append(np.random.uniform(-rng, rng) * n if rng else 0)
    if gen.zoom_range[0] == 1 and gen.zoom_range[1] == 1:
        zoom = (1, 1, 1)
    else:
        zoom = tuple(np.random.uniform(gen.zoom_range[0], gen.zoom_range[1], 3))
    channel = None
    if gen.channel_shift_range != 0:
        channel = [np.random.uniform(-gen.channel_shift_range, gen.channel_shift_range) for _ in range(channels)]
    flips = [False, False, False]         # array axes 0, 1, 2
    for axis, on in ((1, gen.horizontal_flip), (0, gen.vertical_flip), (2, gen.depth_flip)):
        if on and np.random.random() < 0.5:
            flips[axis] = True
    return {"theta": theta, "shift": tuple(shifts), "zoom": zoom, "channel_shift": channel, "flips": tuple(flips)}


def compose_matrix(draw, shape):
    """the centred 4x4 float64 matrix of one draw, built with the reference's numpy calls and ``np.dot`` grouping
    (``np.dot`` of 4x4 float64 goes through BLAS, whose last bits a restated formula would not reproduce)"""
    tx_, ty_, tz_ = draw["theta"]
    rx = np.array([[1, 0, 0, 0], [0, np.cos(tx_), -np.sin(tx_), 0], [0, np.sin(tx_), np.cos(tx_), 0], [0, 0, 0, 1]])
    ry = np.array([[np.cos(ty_), 0, np.sin(ty_), 0], [0, 1, 0, 0], [-np.sin(ty_), 0, np.cos(ty_), 0], [0, 0, 0, 1]])
    rz = np.array([[np.cos(tz_), -np.sin(tz_), 0, 0], [np.sin(tz_), np.cos(tz_), 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    sx, sy, sz = draw["shift"]
    translation = np.array([[1, 0, 0, sx], [0, 1, 0, sy], [0, 0, 1, sz], [0, 0, 0, 1]])
    zx, zy, zz = draw["zoom"]
    zoom = np.array([[zx, 0, 0, 0], [0, zy, 0, 0], [0, 0, zz, 0], [0, 0, 0, 1]])
    m = np.dot(np.dot(rx, ry), rz)
    m = np.dot(np.dot(m, translation), zoom)
    o = [float(n) / 2 + 0.5 for n in shape]            # Keras' centre, not (n - 1) / 2
    offset = np.array([[1, 0, 0, o[0]], [0, 1, 0, o[1]], [0, 0, 1, o[2]], [0, 0, 0, 1]])
    reset = np.array([[1, 0, 0, -o[0]], [0, 1, 0, -o[1]], [0, 0, 1, -o[2]], [0, 0, 0, 1]])
    return np.dot(np.dot(offset, m), reset)


def flip_bits(flips) -> int:
    """(axis 0, axis 1, axis 2) flags -> the ``flip`` bits of ``b200seg_aug3d_param``"""
    return sum(1 << a for a, f in enumerate(flips) if f)


def rescale_form(rescale):
    """``standardize``'s ``x *= rescale`` on an fp32 sample -> (B200SEG_RESCALE_*, value).  numpy (NEP 50) multiplies
    in fp32 by fp32(rescale) for a Python number or an fp32 scalar, and in fp64 (rounded once) for a numpy float64."""
    if not rescale:
        return RESCALE_NONE, 0.0
    rt = np.result_type(np.float32, rescale)
    if rt == np.float32:
        return RESCALE_F32, float(rescale)
    if rt == np.float64:
        return RESCALE_F64, float(rescale)
    raise NotImplementedError(f"rescale of type {type(rescale).__name__} (numpy multiplies in {rt})")


def param_entry(draw, shape):
    """one draw -> the (3x3, offset, channel shifts, flip bits) entry of ``aug3d_param_table``"""
    m4 = compose_matrix(draw, shape)
    shifts = [float(np.float32(u)) for u in draw["channel_shift"]] if draw["channel_shift"] is not None else []
    return m4[:3, :3].reshape(-1), m4[:3, 3], shifts, flip_bits(draw["flips"])


def _current_device():
    return torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")


# ---------------------------------------------------------------------------------------------- the generator
class ImageDataGenerator3D(object):
    """``ImageDataGenerator3D`` of the reference: same constructor, ``random_transform``, ``standardize`` and
    ``flow``; the warp runs on the current CUDA device.  ``transform_batch`` is the per-training-step form."""

    def __init__(self, featurewise_center=False, samplewise_center=False, featurewise_std_normalization=False,
                 samplewise_std_normalization=False, zca_whitening=False, rotation_range=0., width_shift_range=0.,
                 height_shift_range=0., depth_shift_range=0., zoom_range=0., channel_shift_range=0.,
                 fill_mode='nearest', cval=0., horizontal_flip=False, vertical_flip=False, depth_flip=False,
                 rescale=None, preprocessing_function=None, dim_ordering='tf'):
        if featurewise_center or featurewise_std_normalization or zca_whitening:
            raise NotImplementedError("featurewise_* and zca_whitening need statistics the reference never computes "
                                      "(it has no fit())")
        if samplewise_center or samplewise_std_normalization:
            raise NotImplementedError("samplewise_* normalisation is not supported (DataAug3D never sets it)")
        if dim_ordering not in {'tf', 'th'}:
            raise ValueError('dim_ordering should be "tf" (channel after row and column) or "th" (channel before row '
                             'and column). Received arg: ', dim_ordering)
        if dim_ordering == 'th':
            raise NotImplementedError("dim_ordering='th' (the reference leaves its axes unset and fails later)")
        if fill_mode not in AUG_MODES:
            raise NotImplementedError(f"fill_mode {fill_mode!r}: one of {sorted(AUG_MODES)}")
        self.featurewise_center = featurewise_center
        self.samplewise_center = samplewise_center
        self.featurewise_std_normalization = featurewise_std_normalization
        self.samplewise_std_normalization = samplewise_std_normalization
        self.zca_whitening = zca_whitening
        self.rotation_range = rotation_range
        self.width_shift_range = width_shift_range
        self.height_shift_range = height_shift_range
        self.depth_shift_range = depth_shift_range
        self.channel_shift_range = channel_shift_range
        self.fill_mode = fill_mode
        self.cval = cval
        self.horizontal_flip = horizontal_flip
        self.vertical_flip = vertical_flip
        self.depth_flip = depth_flip
        self.rescale = rescale
        self.preprocessing_function = preprocessing_function
        self.dim_ordering = dim_ordering
        self.mean = None
        self.std = None
        self.principal_components = None
        self.channel_axis, self.row_axis, self.col_axis, self.depth_axis = 4, 1, 2, 3
        if np.isscalar(zoom_range):
            self.zoom_range = [1 - zoom_range, 1 + zoom_range]
        elif len(zoom_range) == 2:
            self.zoom_range = [zoom_range[0], zoom_range[1]]
        else:
            raise ValueError('zoom_range should be a float or a tuple or list of two floats. Received arg: ',
                             zoom_range)

    # ------------------------------------------------------------------ reference API
    def flow(self, X, y=None, batch_size=32, shuffle=True, seed=None):
        return NumpyArrayIterator(X, y, self, batch_size=batch_size, shuffle=shuffle, seed=seed,
                                  dim_ordering=self.dim_ordering)

    def standardize(self, x):
        """``x *= rescale`` in place, as the reference (the other options are refused at construction)"""
        if self.rescale:
            x *= self.rescale
        return x

    def random_transform(self, x, y):
        """x numpy fp32 (D, H, W, C), C in {1, 3, 4}; y uint8 / fp32 (D, H, W, 1) -> the reference's (x, y): the warp,
        channel shift and flips (no rescale: that is ``standardize``)"""
        x = np.asarray(x)
        y = np.asarray(y)
        self._check_sample(x, y)
        draw = draw_transform(self, x.shape[:3], x.shape[3])
        xo, yo = self._warp_host_batch(x[None], y[None, ..., 0], [param_entry(draw, x.shape[:3])], rescale=False)
        return xo[0], yo[0][..., None]

    # ------------------------------------------------------------------ per training step
    def transform_batch(self, x, y):
        """x fp32 (N, 1, D, H, W) and y uint8 (N, D, H, W) device tensors -> (fp32 (N, 1, D, H, W), int64
        (N, D, H, W) with y != 0 -> 1, the trainer's binarisation, model/modelVNet.py:576).  Each sample gets fresh
        draws in the reference's per-sample order (as ``flow`` does, ``standardize``'s rescale included); the draw
        table goes up in one small copy and the batch is warped by one launch, on the current stream."""
        if x.dim() != 5 or x.shape[1] != 1 or x.dtype != torch.float32:
            raise ValueError(f"x must be fp32 (N, 1, D, H, W), got {x.dtype} {tuple(x.shape)}")
        if y.dtype != torch.uint8 or tuple(y.shape) != (x.shape[0],) + tuple(x.shape[2:]):
            raise ValueError(f"y must be uint8 (N, D, H, W) matching x, got {y.dtype} {tuple(y.shape)}")
        n, shape = x.shape[0], tuple(int(s) for s in x.shape[2:])
        entries = [param_entry(draw_transform(self, shape, 1), shape) for _ in range(n)]
        be = runtime.get_backend(x)
        xc = x.contiguous()
        yc = y.contiguous()
        xo = torch.empty_like(xc)
        yo = torch.empty(yc.shape, dtype=torch.int64, device=x.device)
        self._launch(be, xc.view(n, *shape, 1), yc, entries, xo.view(n, *shape, 1), yo, rescale=True, binarize=True)
        return xo, yo

    # ------------------------------------------------------------------ plumbing
    @staticmethod
    def _check_sample(x, y):
        if x.ndim != 4 or x.shape[3] not in (1, 3, 4):
            raise ValueError(f"x must be (D, H, W, C) with C in {{1, 3, 4}}, got {x.shape}")
        if x.dtype != np.float32:
            raise TypeError(f"x must be float32 (flow converts), got {x.dtype}")
        if y.shape != x.shape[:3] + (1,):
            raise NotImplementedError(f"y must be (D, H, W, 1) with x's spatial shape, got {y.shape} for x {x.shape}")
        if y.dtype not in (np.uint8, np.float32):
            raise TypeError(f"y must be uint8 or float32, got {y.dtype}")

    def _launch(self, be, x, y, entries, xo, yo, rescale, binarize=False):
        """one batch on the device: x (N, D, H, W, C) fp32, y (N, D, H, W), ``entries`` the N param entries"""
        n = x.shape[0]
        shift = self.channel_shift_range != 0
        table = torch.frombuffer(bytearray(aug3d_param_table(entries)), dtype=torch.uint8)
        if x.is_cuda:
            table = table.pin_memory()
        params = table.to(x.device, non_blocking=True)
        ws = be.augment3d_workspace(n, x.shape[1:4], x.device) if shift else None
        mode, value = rescale_form(self.rescale) if rescale else (RESCALE_NONE, 0.0)
        be.augment3d(x, y, params, xo, yo, mode=AUG_MODES[self.fill_mode], cval=float(self.cval), shift=shift,
                     rescale=value, rescale_mode=mode, binarize=binarize, ws=ws)

    def _warp_host_batch(self, x, y, entries, rescale):
        """numpy (N, D, H, W, C) fp32 and (N, D, H, W) labels -> numpy outputs of the same dtypes: one upload, one
        launch, one download"""
        dev = _current_device()
        xd = torch.from_numpy(np.ascontiguousarray(x)).to(dev)
        yd = torch.from_numpy(np.ascontiguousarray(y)).to(dev)
        be = runtime.get_backend(xd)
        xo = torch.empty_like(xd)
        yo = torch.empty_like(yd)
        self._launch(be, xd, yd, entries, xo, yo, rescale=rescale)
        return xo.cpu().numpy(), yo.cpu().numpy()


class NumpyArrayIterator(object):
    """The reference's ``NumpyArrayIterator`` (and its ``Iterator`` base): same index walk (``np.random.seed(seed +
    total_batches_seen)`` before each batch when seeded, ``np.random.permutation`` at each epoch start when shuffling,
    a short last batch) and float64 batches; each batch's draws are made on the host in the reference's per-sample
    order, then the batch is warped in one launch."""

    def __init__(self, x, y, image_data_generator, batch_size=32, shuffle=False, seed=None, dim_ordering='tf'):
        if y is not None and len(x) != len(y):
            raise ValueError('X (images tensor) and y (labels) should have the same length. Found: X.shape = %s, '
                             'y.shape = %s' % (np.asarray(x).shape, np.asarray(y).shape))
        self.x = np.asarray(x, dtype=np.float32)
        if self.x.ndim != 5:
            raise ValueError('Input data in `NumpyArrayIterator` should have rank 5. You passed an array with shape',
                             self.x.shape)
        if self.x.shape[4] not in {1, 3, 4}:
            raise ValueError('NumpyArrayIterator is set to use the dimension ordering convention "tf" (channels on '
                             'axis 4), i.e. expected either 1, 3 or 4 channels on axis 4. However, it was passed an '
                             'array with shape ' + str(self.x.shape) + ' (' + str(self.x.shape[4]) + ' channels).')
        self.y = np.asarray(y) if y is not None else None
        self.image_data_generator = image_data_generator
        self.dim_ordering = dim_ordering
        self.n = self.x.shape[0]
        self.batch_size = batch_size
        self.shuffle = shuffle
        self.batch_index = 0
        self.total_batches_seen = 0
        self.lock = threading.Lock()
        self.index_generator = self._flow_index(self.n, batch_size, shuffle, seed)

    def reset(self):
        self.batch_index = 0

    def _flow_index(self, n, batch_size=32, shuffle=False, seed=None):
        self.reset()
        while 1:
            if seed is not None:
                np.random.seed(seed + self.total_batches_seen)
            if self.batch_index == 0:
                index_array = np.arange(n)
                if shuffle:
                    index_array = np.random.permutation(n)
            current_index = (self.batch_index * batch_size) % n
            if n >= current_index + batch_size:
                current_batch_size = batch_size
                self.batch_index += 1
            else:
                current_batch_size = n - current_index
                self.batch_index = 0
            self.total_batches_seen += 1
            yield index_array[current_index: current_index + current_batch_size], current_index, current_batch_size

    def __iter__(self):
        return self

    def __next__(self, *args, **kwargs):
        return self.next(*args, **kwargs)

    def next(self):
        with self.lock:
            index_array, _, current_batch_size = next(self.index_generator)
        gen = self.image_data_generator
        xb = self.x[index_array]
        yb = self.y[index_array].astype(np.float32)
        if yb.shape[1:] != xb.shape[1:4] + (1,):
            raise NotImplementedError(f"labels must be (N, D, H, W, 1) with the images' spatial shape, got "
                                      f"{self.y.shape} for {self.x.shape}")
        shape = xb.shape[1:4]
        entries = [param_entry(draw_transform(gen, shape, xb.shape[4]), shape) for _ in range(current_batch_size)]
        xo, yo = gen._warp_host_batch(xb, yb[..., 0], entries, rescale=True)
        return xo.astype(np.float64), yo[..., None].astype(np.float64)
