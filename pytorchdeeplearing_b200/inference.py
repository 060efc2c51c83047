"""Forward-only inference path (SURVEY.md 8f-3): ``predict`` of the reference wrappers
(model/modelVNet.py:655-676, model/modelUnet.py:641-662), the sliding-window ``inference_patch``
(model/modelUnet.py:707-763) on the drop-in networks, and the whole-volume 3-D ``XModel.inference`` /
``inference_patch`` chains with their SimpleITK resamples and intensity normalisations on the device
(``inference3d``, ``inference_patch3d``, ``resample3d``; csrc/resample.cu), and the 2-D ``XModel.inference`` with its
bit-exact cv2 bilinear resizes (``inference2d``, ``resize2d``; csrc/resize2d.cu).

The reference runs the net, copies the fp32 probabilities to the host and thresholds / arg-maxes them with numpy.
Here the head kernel writes the uint8 mask directly (``b200seg_head_mask``: neither logits nor probs are
materialised) and only the mask crosses PCIe (1 byte per voxel instead of 4*C).
"""
from __future__ import annotations

from typing import Sequence

import numpy as np
import torch

from . import runtime
from ._abi import NORM_MEANSTD, NORM_NONE, NORM_PCTL, resize_src_table
from .engine import Engine


def _require_segmenter(model) -> None:
    if getattr(model, "_arch", None) == "resnet":
        raise TypeError(f"{type(model).__name__} is a classifier: it has no segmentation mask to predict; call the "
                        "model itself for its (N, numclass) logits, as the reference's ResNet predict does")


@torch.no_grad()
def predict_mask(model, x: torch.Tensor, out_threshold: float = 0.5) -> torch.Tensor:
    """x (N, Cin, [D,] H, W) on the model's device -> uint8 mask (N, [D,] H, W): ``(sigmoid > out_threshold) * 255``
    for a one-class head, ``argmax`` over the classes otherwise (model/modelVNet.py:668-675).  Eval-mode forward.
    Segmentation nets only: a classifier (ResNet2d / ResNet3d) raises ``TypeError``."""
    _require_segmenter(model)
    be = runtime.get_backend(x)
    eng = Engine(be, runtime.act_dtype(), model._dims)
    eng.mask_threshold = float(out_threshold)
    P = dict(zip(model._pnames, [p.detach() for _, p in model.named_parameters()]))
    xx = x.detach()
    if xx.dtype != torch.float32:
        xx = xx.float()
    mask, _ = getattr(eng, model._arch + "_forward")(P, xx, None, False)
    return mask


def predict(model, full_img, out_threshold: float = 0.5) -> np.ndarray:
    """``XModel.predict(full_img, out_threshold)`` (model/modelVNet.py:655-676): numpy image (Cin, [D,] H, W) ->
    numpy uint8 mask ([D,] H, W)."""
    _require_segmenter(model)
    dev = next(model.parameters()).device
    img = torch.as_tensor(np.ascontiguousarray(full_img)).float().unsqueeze(0).to(dev)
    was_training = model.training
    model.eval()
    try:
        mask = predict_mask(model, img, out_threshold)
    finally:
        model.train(was_training)
    return mask[0].cpu().numpy().astype(np.uint8)


def _starts(size: int, patch: int, step: int):
    """window origins along one axis: stride ``step``, the last window clamped to the volume end"""
    if size <= patch:
        return [0]
    s = list(range(0, size - patch + 1, step))
    if s[-1] != size - patch:
        s.append(size - patch)
    return s


@torch.no_grad()
def sliding_window_mask(model, image, patch_size: Sequence[int], step: Sequence[int] = None, batch: int = 4,
                        out_threshold: float = 0.5) -> np.ndarray:
    """``inference_patch`` (model/modelUnet.py:707-763) without the SimpleITK resampling around it: tile the volume
    (Cin, D, H, W) [or image (Cin, H, W)] with ``patch_size`` windows every ``step`` voxels (default: half a patch, as
    the reference), predict ``batch`` windows per forward on the device, accumulate the masks on the device and
    binarise the union (``out_mask[out_mask != 0] = 1``).  Only the final uint8 volume is copied to the host."""
    _require_segmenter(model)
    dev = next(model.parameters()).device
    vol = torch.as_tensor(np.ascontiguousarray(image)).float().to(dev)
    return _window_union(model, vol, patch_size, step, batch, out_threshold).cpu().numpy()


@torch.no_grad()
def _window_union(model, vol: torch.Tensor, patch_size, step, batch, out_threshold) -> torch.Tensor:
    """the device part of ``sliding_window_mask``: fp32 ``vol`` on the model's device -> uint8 union on the device"""
    dev = vol.device
    dims = model._dims
    if vol.dim() != dims + 1:
        raise ValueError(f"expected (Cin, {'D, ' if dims == 3 else ''}H, W), got {tuple(vol.shape)}")
    patch = tuple(int(p) for p in patch_size)
    step = tuple(int(s) for s in step) if step is not None else tuple(max(1, p // 2) for p in patch)
    sp = tuple(vol.shape[1:])
    if any(s < p for s, p in zip(sp, patch)):
        raise ValueError(f"volume {sp} is smaller than the patch {patch}")
    origins = [()]
    for size, p, s in zip(sp, patch, step):
        origins = [o + (a,) for o in origins for a in _starts(size, p, s)]
    acc = torch.zeros(sp, dtype=torch.int32, device=dev)
    was_training = model.training
    model.eval()
    try:
        for i in range(0, len(origins), batch):
            chunk = origins[i:i + batch]
            xb = torch.stack([vol[(slice(None),) + tuple(slice(a, a + p) for a, p in zip(o, patch))] for o in chunk])
            mb = predict_mask(model, xb, out_threshold)
            for o, m in zip(chunk, mb):
                acc[tuple(slice(a, a + p) for a, p in zip(o, patch))] += m.to(torch.int32)
    finally:
        model.train(was_training)
    return (acc != 0).to(torch.uint8)


# ---------------------------------------------------------------------------------------- whole-volume 3-D inference
_INTENSITY = {None: NORM_NONE, "vnet": NORM_MEANSTD, "unet": NORM_PCTL}
_VOLUME_DTYPES = (np.uint8, np.int16, np.int32, np.float32)


def _is_sitk(image) -> bool:
    return all(hasattr(image, a) for a in ("GetSize", "GetSpacing", "GetOrigin", "GetDirection"))


def _volume(image, spacing=None):
    """numpy (D, H, W) or SimpleITK image -> (contiguous numpy volume, spacing (x, y, z) or None, geometry or None)"""
    geom = None
    if _is_sitk(image):
        import SimpleITK as sitk
        geom = (tuple(image.GetOrigin()), tuple(image.GetSpacing()), tuple(image.GetDirection()))
        if spacing is None:
            spacing = geom[1]
        arr = sitk.GetArrayFromImage(image)
    else:
        arr = image
    arr = np.ascontiguousarray(arr)
    if arr.ndim != 3:
        raise ValueError(f"expected a (D, H, W) volume, got shape {arr.shape}")
    if arr.dtype not in _VOLUME_DTYPES:
        raise TypeError(f"volumes must be uint8, int16, int32 or float32, got {arr.dtype}")
    if spacing is not None:
        spacing = tuple(float(s) for s in spacing)
        if len(spacing) != 3 or not all(np.isfinite(s) and s > 0 for s in spacing):
            raise ValueError(f"spacing must be three positive numbers, got {spacing}")
    return arr, spacing, geom


def _as_result(mask: np.ndarray, geom):
    """the mask as a SimpleITK image with the input's geometry when the input was one"""
    if geom is None:
        return mask
    import SimpleITK as sitk
    img = sitk.GetImageFromArray(mask)
    img.SetOrigin(geom[0])
    img.SetSpacing(geom[1])
    img.SetDirection(geom[2])
    return img


def _size_xyz(size, what):
    s = tuple(int(v) for v in size)
    if len(s) != 3 or min(s) < 1:
        raise ValueError(f"{what} must be three sizes >= 1 (x, y, z), got {tuple(size)}")
    return s


def spacing_size(size_xyz, spacing, new_spacing):
    """``resize_image_itk``'s output size (dataprocess/utils.py:132-135): (size / (new_spacing / spacing)).astype(int),
    all (x, y, z)"""
    factor = np.array(new_spacing, float) / np.array(spacing, float)
    return tuple(int(v) for v in (np.array(size_xyz) / factor).astype(np.int64))


def _check_intensity(intensity):
    if intensity not in _INTENSITY:
        raise ValueError(f"intensity must be 'vnet', 'unet' or None, got {intensity!r}")
    return _INTENSITY[intensity]


def _network_input(be, vol: torch.Tensor, out_zyx, ratio_zyx, mode, window):
    """device volume (D, H, W) -> (fp32 network input (1, 1, oD, oH, oW), resample workspace or None)"""
    x = torch.empty(out_zyx, dtype=torch.float32, device=vol.device)
    if mode == NORM_NONE:
        be.resample_linear(vol, ratio_zyx, x)
        return x.view((1, 1) + tuple(out_zyx)), None
    ws = be.resample_workspace(mode, out_zyx, vol.device)
    lower, upper = (float(w) for w in window)
    be.resample_linear(vol, ratio_zyx, x, mode, lower, upper, ws)
    xn = torch.empty_like(x)
    be.normalize(mode, x, ws, xn)
    return xn.view((1, 1) + tuple(out_zyx)), ws


def _require_3d(model):
    _require_segmenter(model)
    if model._dims != 3:
        raise ValueError(f"{type(model).__name__} is a 2-D network; the whole-volume inference is 3-D")


@torch.no_grad()
def _inference3d_device(model, vol: torch.Tensor, newSize, mode, out_threshold, window) -> torch.Tensor:
    """device volume (D, H, W) -> device uint8 mask (D, H, W); no host synchronisation"""
    be = runtime.get_backend(vol)
    in_zyx = tuple(vol.shape)
    out_zyx = tuple(reversed(_size_xyz(newSize, "newSize")))
    x, _ = _network_input(be, vol, out_zyx, [a / b for a, b in zip(in_zyx, out_zyx)], mode, window)
    was_training = model.training
    model.eval()
    try:
        m = predict_mask(model, x, out_threshold)[0].contiguous()
    finally:
        model.train(was_training)
    out = torch.empty(in_zyx, dtype=torch.uint8, device=vol.device)
    be.resample_nearest_u8(m, [a / b for a, b in zip(out_zyx, in_zyx)], in_zyx, out)
    return out


def inference3d(model, image, newSize=(96, 96, 96), intensity="vnet", out_threshold: float = 0.5,
                window=(-100.0, 100.0)):
    """``XModel.inference(imagesitk, newSize)`` (model/modelVNet.py:678-698, model/modelUnet.py:684-705) of a 3-D
    segmentation net: linear resample of ``image`` to ``newSize`` (x, y, z), intensity normalisation, ``predict``,
    and the nearest-neighbour resample of the uint8 mask back to the image's grid.

    ``image``: a numpy (D, H, W) volume (uint8, int16, int32 or float32) -> numpy uint8 mask (D, H, W); or a SimpleITK
    image -> SimpleITK uint8 mask with the image's origin, spacing and direction.  ``intensity``: ``"vnet"``
    (``ConvertitkTrunctedValue(.., upper, lower, 'meanstd')``: truncate to ``window`` = (lower, upper), then z-score
    with the N - 1 deviation; the VNet3d models), ``"unet"`` (``normalize()``: 5/95 percentile clip, z-score of the
    nonzero voxels; the UNet3d models) or None (no normalisation; no reference method does this).  Only the raw volume (in its own dtype) goes to the device and only the final mask comes back."""
    _require_3d(model)
    mode = _check_intensity(intensity)
    _size_xyz(newSize, "newSize")
    arr, _, geom = _volume(image)
    dev = next(model.parameters()).device
    vol = torch.from_numpy(arr).to(dev)
    mask = _inference3d_device(model, vol, newSize, mode, out_threshold, window)
    return _as_result(mask.cpu().numpy(), geom)


@torch.no_grad()
def _inference_patch3d_device(model, vol: torch.Tensor, spacing, newSpacing, patch_size, mode, window, batch,
                              out_threshold) -> torch.Tensor:
    be = runtime.get_backend(vol)
    in_zyx = tuple(vol.shape)
    size_xyz = tuple(reversed(in_zyx))
    rs_xyz = spacing_size(size_xyz, spacing, newSpacing)
    if min(rs_xyz) < 1:
        raise ValueError(f"new spacing {tuple(newSpacing)} leaves an empty grid {rs_xyz}")
    rs_zyx = tuple(reversed(rs_xyz))
    patch_zyx = tuple(reversed(_size_xyz(patch_size, "patch_size")))
    if any(s < p for s, p in zip(rs_zyx, patch_zyx)):
        raise ValueError(f"resampled volume {rs_xyz} is smaller than the patch {tuple(patch_size)} (x, y, z)")
    fwd = [n / o for n, o in zip(reversed(newSpacing), reversed(spacing))]
    x, _ = _network_input(be, vol, rs_zyx, fwd, mode, window)
    # the reference's loops multiply the window index by the patch size (modelUnet.py:723-734), so windows start every
    # p * (p // 2) voxels, the last one clamped to the end
    step = tuple(p * (p // 2) for p in patch_zyx)
    union = _window_union(model, x[0], patch_zyx, step, batch, out_threshold).contiguous()
    back_zyx = tuple(reversed(spacing_size(rs_xyz, newSpacing, spacing)))
    out = torch.empty(in_zyx, dtype=torch.uint8, device=vol.device)
    be.resample_nearest_u8(union, [o / n for n, o in zip(reversed(newSpacing), reversed(spacing))], back_zyx, out)
    return out


def inference_patch3d(model, image, spacing=None, newSpacing=(0.5, 0.5, 0.5), patch_size=(96, 96, 96),
                      intensity="vnet", window=(-1024.0, -800.0), batch: int = 4, out_threshold: float = 0.5):
    """``XModel.inference_patch(imagesitk, newSpacing)`` (model/modelUnet.py:707-763): linear resample of ``image``
    from ``spacing`` to ``newSpacing`` (x, y, z; a SimpleITK image brings its own spacing), intensity normalisation
    (default: the reference's ``ConvertitkTrunctedValue(.., -800, -1024, 'meanstd')``), the reference's window walk
    with ``patch_size`` (x, y, z) windows, the binarised union, the nearest-neighbour resample back and the crop / zero
    pad to the image's shape.  Returns a uint8 0/1 mask like ``inference3d``."""
    _require_3d(model)
    mode = _check_intensity(intensity)
    arr, spacing, geom = _volume(image, spacing)
    if spacing is None:
        raise ValueError("a numpy volume needs its spacing (x, y, z)")
    newSpacing = tuple(float(s) for s in newSpacing)
    if len(newSpacing) != 3 or not all(np.isfinite(s) and s > 0 for s in newSpacing):
        raise ValueError(f"newSpacing must be three positive numbers, got {newSpacing}")
    if int(batch) < 1:
        raise ValueError("batch must be >= 1")
    dev = next(model.parameters()).device
    vol = torch.from_numpy(arr).to(dev)
    mask = _inference_patch3d_device(model, vol, spacing, newSpacing, patch_size, mode, window, int(batch),
                                     out_threshold)
    return _as_result(mask.cpu().numpy(), geom)


def resample3d(volume, newSize=None, spacing=None, newSpacing=None, interpolator: str = "linear", out_size=None,
               device="cuda"):
    """The two resamples of the whole-volume inference on their own.  ``volume``: (D, H, W) numpy array or tensor
    (numpy in -> numpy out; a tensor stays on its device).  The output grid is ``newSize`` (x, y, z) with input-index
    step S_in / S_out, or, given ``spacing`` and ``newSpacing``, ``spacing_size(...)`` with step new / old spacing.
    ``interpolator="linear"``: uint8 / int16 / int32 / float32 input -> float32 values of the input's pixel type.
    ``"nearest"``: uint8 input -> uint8, placed in the corner of an ``out_size`` (x, y, z) array that is cropped or
    zero-padded (inference_patch's back-resample; default: the resampled size)."""
    if interpolator not in ("linear", "nearest"):
        raise ValueError(f"interpolator must be 'linear' or 'nearest', got {interpolator!r}")
    is_np = not isinstance(volume, torch.Tensor)
    vol = torch.from_numpy(np.ascontiguousarray(volume)) if is_np else volume.contiguous()
    if is_np:
        vol = vol.to(device)
    if vol.dim() != 3:
        raise ValueError(f"expected a (D, H, W) volume, got shape {tuple(vol.shape)}")
    in_zyx = tuple(vol.shape)
    if (newSize is None) == (newSpacing is None):
        raise ValueError("give either newSize or (spacing, newSpacing)")
    if newSize is not None:
        out_xyz = _size_xyz(newSize, "newSize")
        ratio = [a / b for a, b in zip(in_zyx, reversed(out_xyz))]
    else:
        if spacing is None:
            raise ValueError("newSpacing needs the volume's spacing")
        sp = tuple(float(s) for s in spacing)
        nsp = tuple(float(s) for s in newSpacing)
        if len(sp) != 3 or len(nsp) != 3 or not all(np.isfinite(s) and s > 0 for s in sp + nsp):
            raise ValueError("spacings must be three positive numbers")
        out_xyz = spacing_size(tuple(reversed(in_zyx)), sp, nsp)
        if min(out_xyz) < 1:
            raise ValueError(f"new spacing {nsp} leaves an empty grid {out_xyz}")
        ratio = [n / o for n, o in zip(reversed(nsp), reversed(sp))]
    be = runtime.get_backend(vol)
    if interpolator == "linear":
        if vol.dtype not in (torch.uint8, torch.int16, torch.int32, torch.float32):
            raise TypeError(f"volumes must be uint8, int16, int32 or float32, got {vol.dtype}")
        out = torch.empty(tuple(reversed(out_xyz)), dtype=torch.float32, device=vol.device)
        be.resample_linear(vol, ratio, out)
    else:
        if vol.dtype != torch.uint8:
            raise TypeError(f"the nearest-neighbour resample takes uint8 masks, got {vol.dtype}")
        full = tuple(reversed(_size_xyz(out_size, "out_size"))) if out_size is not None else tuple(reversed(out_xyz))
        out = torch.empty(full, dtype=torch.uint8, device=vol.device)
        be.resample_nearest_u8(vol, ratio, tuple(reversed(out_xyz)), out)
    return out.cpu().numpy() if is_np else out


# ---------------------------------------------------------------------------------------- 2-D image resize and inference
MAX_RESIZE_BATCH = 65535


def resize_desc(be, entries, device) -> torch.Tensor:
    """[(byte offset, h, w)] of a ragged uint8 batch -> the int64 [N, 2] device table of ``b200seg_resize_src``
    (uploaded through kernel arguments: no copy from pageable memory, no host synchronisation)"""
    if not 1 <= len(entries) <= MAX_RESIZE_BATCH:
        raise ValueError(f"a resize batch holds 1 to {MAX_RESIZE_BATCH} images, got {len(entries)}")
    raw = resize_src_table(entries)
    return be.upload_bytes(raw, device)[:len(raw)].view(torch.int64).view(len(entries), 2)


def _dsize(dsize):
    d = tuple(int(v) for v in dsize)
    if len(d) != 2 or min(d) < 1:
        raise ValueError(f"dsize must be (width, height) >= 1, got {tuple(dsize)}")
    return d


def resize2d(image, dsize, device="cuda"):
    """``cv2.resize(image, dsize)`` with its default INTER_LINEAR, bit for bit (csrc/resize2d.cu).  ``dsize`` is
    (width, height), as in cv2.  ``image``: uint8 (H, W) or a batch (N, H, W), as a numpy array (-> numpy, computed on
    ``device``) or a tensor (-> a tensor on the tensor's device).  Returns uint8 (height, width) or (N, height, width)."""
    is_np = not isinstance(image, torch.Tensor)
    img = torch.from_numpy(np.ascontiguousarray(image)) if is_np else image
    if img.dtype != torch.uint8:
        raise TypeError(f"resize2d takes uint8 images, got {img.dtype}")
    if img.dim() not in (2, 3):
        raise ValueError(f"expected an (H, W) image or an (N, H, W) batch, got shape {tuple(img.shape)}")
    if min(img.shape) < 1:
        raise ValueError(f"image sizes must be >= 1, got {tuple(img.shape)}")
    ow, oh = _dsize(dsize)
    batch = img if img.dim() == 3 else img.unsqueeze(0)
    if is_np:
        batch = batch.to(device)
    batch = batch.contiguous()
    n, h, w = batch.shape
    be = runtime.get_backend(batch)
    out = torch.empty((n, oh, ow), dtype=torch.uint8, device=batch.device)
    be.resize_linear(batch.view(-1), resize_desc(be, [(i * h * w, h, w) for i in range(n)], batch.device), out)
    if img.dim() == 2:
        out = out[0]
    return out.cpu().numpy() if is_np else out


@torch.no_grad()
def _inference2d_device(model, src: torch.Tensor, newSize, out_threshold) -> torch.Tensor:
    """device uint8 image (h, w) -> device uint8 mask (w, h), or the uint8 class value (1,) of a classifier; no host
    synchronisation"""
    be = runtime.get_backend(src)
    dev = src.device
    h, w = src.shape
    W, H = _dsize(newSize)
    x = torch.empty((1, H, W), dtype=torch.float32, device=dev)
    be.resize_linear(src.reshape(-1), resize_desc(be, [(0, h, w)], dev), x)       # cv2.resize, then / 255.
    x = x.view(1, 1, H, W)
    was_training = model.training
    model.eval()
    try:
        if getattr(model, "_arch", None) == "resnet":
            logits = model(x).contiguous()                  # (1, numclass) fp32
            cls = torch.empty((1,), dtype=torch.uint8, device=dev)
            be.mask_logits(logits, float(out_threshold), cls)
            return cls
        m = predict_mask(model, x, out_threshold)[0].contiguous()
    finally:
        model.train(was_training)
    # cv2.resize(out_mask, image.shape): image.shape = (h, w) is read as (width, height)
    out = torch.empty((1, w, h), dtype=torch.uint8, device=dev)
    be.resize_linear(m.view(-1), resize_desc(be, [(0, H, W)], dev), out)
    return out[0]


def inference2d(model, image, newSize=(512, 512), out_threshold: float = 0.5):
    """``XModel.inference(image)`` of a 2-D network (model/modelVNet.py:231-242,450-461, model/modelUnet.py:231-242,
    450-461, model/modelResNet.py:212-221,428-437): ``cv2.resize(image, newSize)``, ``/ 255.``, ``predict``, and for a
    segmentation net ``cv2.resize(out_mask, image.shape)``.  ``image``: uint8 (H, W), the output of
    ``cv2.imread(path, 0)``; ``newSize``: the wrapper's (image_width, image_height).  Only the raw bytes go to the
    device and only the result comes back; both resizes are bit-exact cv2 INTER_LINEAR.

    Segmentation nets (VNet2d, UNet2d) return a uint8 numpy mask with the reference's two quirks kept: the mask is
    resized bilinearly (a 0/255 mask gains intermediate values at its edges, class indices are interpolated), and
    ``dsize = image.shape`` is (height, width) read as (width, height), so an (H, W) image gives a (W, H) mask.
    ResNet2d returns what the classifier's ``predict`` returns: a numpy int64, 0 / 255 for one class
    (sigmoid > out_threshold), the arg-max class index otherwise.  3-D networks raise ``ValueError``."""
    if getattr(model, "_dims", None) != 2:
        raise ValueError(f"{type(model).__name__} is a 3-D network; inference2d runs the 2-D networks")
    _dsize(newSize)
    arr = np.ascontiguousarray(image)
    if arr.dtype != np.uint8:
        raise TypeError(f"inference2d takes the uint8 image of cv2.imread(path, 0), got {arr.dtype}")
    if arr.ndim != 2 or min(arr.shape) < 1:
        raise ValueError(f"expected an (H, W) image with sizes >= 1, got shape {arr.shape}")
    dev = next(model.parameters()).device
    out = _inference2d_device(model, torch.from_numpy(arr).to(dev), newSize, out_threshold)
    if getattr(model, "_arch", None) == "resnet":
        return np.int64(out.cpu().numpy()[0])
    return out.cpu().numpy()


__all__ = ["predict_mask", "predict", "sliding_window_mask", "inference3d", "inference_patch3d", "resample3d",
           "spacing_size", "resize2d", "inference2d"]
