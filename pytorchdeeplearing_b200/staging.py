"""Device-side input staging: the per-sample host work of the reference's 2-D dataset, done on the GPU.

Reference: ``datasetModelSegwithopencv.__getitem__`` (model/dataset.py:128-158) z-scores every 8-bit image on the host
in float64 (``(image - image.mean()) / image.std()``), converts it to fp32 (4 B/pixel) and the label to int64
(8 B/pixel); the trainer then binarises the label (``y[y != 0] = 1``, model/modelUnet.py:130) and copies both to the
device (``:132``).  Here the raw uint8 image and label batches (1 B/pixel each) are copied from pinned host memory and
normalised / widened by two small kernels (csrc/staging.cu), on a side stream, one batch ahead of the step that consumes
them.  With ``max_source_pixels`` the datasets' ``cv2.resize`` (dataset.py:63,140,154) runs on the device too: the
images (and labels) of a batch may have any sizes, they are packed into one pinned ragged buffer, sent with one copy,
resized bit for bit as cv2's INTER_LINEAR (csrc/resize2d.cu) and then staged by the same two kernels.  File reading and
``cv2.imread`` stay on the host; the 3-D dataset (``datasetModelSegwithnpy``, dataset.py:82-117) loads volumes that
``DataAug3D`` augmented offline and needs no arithmetic itself; that augmentation runs on the device through
``ImageDataGenerator3D`` (augment.py), offline or per step with ``transform_batch``.

    stager = InputStager(device, (8, 512, 512))
    stager.put(images_u8, labels_u8)           # host uint8 arrays/tensors [N, H, W]; returns immediately
    x, y = stager.get()                        # x [N, 1, H, W] fp32, y [N, H, W] int64, ordered after the current stream

    stager = InputStager(device, (8, 512, 512), max_source_pixels=8 * 1024 * 1024)
    stager.put([cv2.imread(p, 0) for p in paths], [cv2.imread(p, 0) for p in label_paths])   # any sizes

    stager = InputStager(device, (8, 512, 512), max_source_pixels=8 * 1024 * 1024, augment=Segmenation_Aug())
    stager.put(images, labels)     # + the reference's 2-D augmentation at each source size, before the resize
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import torch

from . import runtime
from ._abi import AUG2D_PARAM_BYTES, RESIZE_SRC_BYTES as _DESC, resize_src_table


class InputStager:
    """Double-buffered uint8 -> (z-scored float image, int64 label) staging for a fixed batch shape [N, *spatial].

    ``max_source_pixels``: resize mode for 2-D batches (shape (N, H, W)).  ``put`` then takes N uint8 images of any,
    possibly different, (h, w) -- at most ``max_source_pixels`` pixels in total, and as many for the labels -- and
    resizes each to (H, W) as ``cv2.resize(img, (W, H))`` before the z-score; labels are resized the same way before
    the widening.  For square targets this is what the reference's ``datasetModelSegwithopencv`` /
    ``datasetModelClassifywithopencv`` return (image, and label after the trainer's binarisation); those classes pass
    (H, W) to cv2 as (width, height), so their own assert refuses a non-square target, which the stager accepts.

    ``augment``: a ``Segmenation_Aug`` (augment2d.py), resize mode only.  ``put`` then draws each image's parameters
    on the host, ships them in the same ragged copy and augments every image (and its label, which must have the
    image's size) at its source size before the resize: the reference's order, where the augmentation writes its files
    offline and the dataset resizes and z-scores what it reads back."""

    def __init__(self, device, shape: Sequence[int], dtype: torch.dtype = torch.float32, binarize_labels: bool = True,
                 slots: int = 2, backend=None, max_source_pixels: Optional[int] = None, augment=None):
        self.device = torch.device(device)
        self.shape = tuple(int(v) for v in shape)
        self.dtype = dtype
        self.binarize = bool(binarize_labels)
        self.be = backend if backend is not None else runtime.get_backend(torch.empty(0, device=self.device))
        self.max_source_pixels = None if max_source_pixels is None else int(max_source_pixels)
        if self.max_source_pixels is not None:
            if len(self.shape) != 3 or min(self.shape) < 1:
                raise ValueError(f"InputStager: the resize mode stages 2-D batches (N, H, W), got shape {self.shape}")
            if self.max_source_pixels < 1:
                raise ValueError("InputStager: max_source_pixels must be >= 1")
        self.augment = augment
        if augment is not None and self.max_source_pixels is None:
            raise ValueError("InputStager: augment needs the resize mode (max_source_pixels)")
        cuda = self.device.type == "cuda"
        self._stream = torch.cuda.Stream(self.device) if cuda else None
        self._slots = []
        for _ in range(max(1, int(slots))):
            if self.max_source_pixels is None:
                h_img = torch.empty(self.shape, dtype=torch.uint8, pin_memory=cuda)
                h_lab = torch.empty(self.shape, dtype=torch.uint8, pin_memory=cuda)
                h_src = d_src = None
            else:
                # one ragged slot: [image descriptors][label descriptors][image pixels, label pixels]
                nb = self._pixel_base() + 2 * self.max_source_pixels
                h_img = h_lab = None
                h_src = torch.empty(nb, dtype=torch.uint8, pin_memory=cuda)
                d_src = torch.empty(nb, dtype=torch.uint8, device=self.device)
            d_img = torch.empty(self.shape, dtype=torch.uint8, device=self.device)
            d_lab = torch.empty(self.shape, dtype=torch.uint8, device=self.device)
            x = torch.empty((self.shape[0], 1) + self.shape[1:], dtype=dtype, device=self.device)
            y = torch.empty(self.shape, dtype=torch.int64, device=self.device)
            ev = torch.cuda.Event() if cuda else None
            self._slots.append(dict(h_img=h_img, h_lab=h_lab, h_src=h_src, d_src=d_src, d_img=d_img, d_lab=d_lab, x=x,
                                    y=y, ready=ev, free=None))
        if augment is not None:                # the augmented images and labels, and the blur workspace
            self._d_aug = torch.empty(2 * self.max_source_pixels, dtype=torch.uint8, device=self.device)
            self._aug_ws = self.be.augment2d_workspace(self._d_aug.numel(), self.device)
        self._put = 0
        self._got = 0
        if self.max_source_pixels is None:
            self.h2d_bytes_per_batch = 2 * int(torch.Size(self.shape).numel())
        else:                                  # an upper bound: a batch sends its descriptors and its own pixels only
            self.h2d_bytes_per_batch = self._pixel_base() + 2 * self.max_source_pixels

    def _pixel_base(self) -> int:
        return (2 * _DESC + (AUG2D_PARAM_BYTES if self.augment is not None else 0)) * self.shape[0]

    def put(self, images, labels=None) -> None:
        """Queue one batch: uint8 images [N, *spatial] (numpy array or tensor) and, optionally, uint8 labels.  In resize
        mode: a length-N sequence of uint8 (h, w) images (and labels) of any sizes."""
        if self._put - self._got >= len(self._slots):
            raise RuntimeError("InputStager: every slot holds a batch that has not been taken (call get())")
        s = self._slots[self._put % len(self._slots)]
        if self.max_source_pixels is not None:
            self._put_ragged(s, images, labels)
            return
        img = torch.as_tensor(images)
        if img.dtype != torch.uint8 or tuple(img.shape) != self.shape:
            raise ValueError(f"InputStager: expected uint8 images of shape {self.shape}, got {img.dtype} {tuple(img.shape)}")
        lab = None
        if labels is not None:
            lab = torch.as_tensor(labels)
            if lab.dtype != torch.uint8 or tuple(lab.shape) != self.shape:
                raise ValueError(f"InputStager: expected uint8 labels of shape {self.shape}, got {lab.dtype} {tuple(lab.shape)}")
        if s["free"] is not None:
            s["free"].synchronize()            # the step that consumed this slot's last batch has finished with it
        s["h_img"].copy_(img)
        if lab is not None:
            s["h_lab"].copy_(lab)
        s["has_labels"] = lab is not None
        self._launch(s, self._run)

    def _launch(self, s, run) -> None:
        if self._stream is None:
            run(s)
        else:
            with torch.cuda.stream(self._stream):
                run(s)
                s["ready"].record(self._stream)
        self._put += 1

    def _run(self, s) -> None:
        s["d_img"].copy_(s["h_img"], non_blocking=True)
        self.be.stage_images_u8(s["d_img"], s["x"])
        if s["has_labels"]:
            s["d_lab"].copy_(s["h_lab"], non_blocking=True)
            self.be.stage_labels_u8(s["d_lab"], s["y"], self.binarize)

    # ------------------------------------------------------------------ resize mode
    def _ragged(self, seq, what):
        """a length-N sequence of uint8 (h, w) images -> list of tensors; raises on a wrong count, dtype or rank"""
        n = self.shape[0]
        items = [torch.as_tensor(t) for t in seq]
        if len(items) != n:
            raise ValueError(f"InputStager: expected {n} {what}, got {len(items)}")
        for t in items:
            if t.dtype != torch.uint8 or t.dim() != 2 or min(t.shape) < 1:
                raise ValueError(f"InputStager: {what} must be uint8 (h, w) arrays with sizes >= 1, got {t.dtype} "
                                 f"{tuple(t.shape)}")
        total = sum(int(t.numel()) for t in items)
        if total > self.max_source_pixels:
            raise ValueError(f"InputStager: the {what} of this batch hold {total} pixels, more than max_source_pixels "
                             f"= {self.max_source_pixels}")
        return items

    def _put_ragged(self, s, images, labels) -> None:
        imgs = self._ragged(images, "images")
        labs = self._ragged(labels, "labels") if labels is not None else []
        if s["free"] is not None:
            s["free"].synchronize()            # the step that consumed this slot's last batch has finished with it
        h, base = s["h_src"], self._pixel_base()
        off, entries = 0, []
        for t in imgs + labs:                  # pixels: images, then labels; offsets from the first image pixel
            k = int(t.numel())
            h[base + off:base + off + k].copy_(t.reshape(-1))
            entries.append((off, t.shape[0], t.shape[1]))
            off += k
        table = resize_src_table(entries)
        if self.augment is not None:
            table = table.ljust(2 * _DESC * len(imgs), b"\0") + self._augment_table(s, imgs, labs, entries)
        h[:len(table)].copy_(torch.frombuffer(bytearray(table), dtype=torch.uint8))
        s["used"] = base + off
        s["has_labels"] = labels is not None
        self._launch(s, self._run_ragged)

    def _augment_table(self, s, imgs, labs, entries) -> bytes:
        """each image's draws -> its ``b200seg_aug2d_param`` bytes; the output goes to the image's own offset of the
        augmented buffer (its label's likewise)"""
        from .augment2d import check_pair, draw_params, param_entry
        n, out, stages = len(imgs), [], 0
        for i, t in enumerate(imgs):
            h, w, _ = check_pair(t, labs[i] if labs else None)
            off = entries[i][0]
            moff = entries[n + i][0] if labs else -1
            # the reference writes 3-channel BMPs that the dataset reads back as gray: MotionBlur's fp32 tail as BGR
            e, f = param_entry(draw_params(), h, w, 1, off, off, moff, max(moff, 0), filter_cn=3)
            out.append(e)
            stages |= f
        s["aug_stages"] = stages
        s["aug_max_hw"] = max(int(t.numel()) for t in imgs)
        return b"".join(out)

    def _run_ragged(self, s) -> None:
        n, base, d = self.shape[0], self._pixel_base(), s["d_src"]
        d[:s["used"]].copy_(s["h_src"][:s["used"]], non_blocking=True)       # descriptors and pixels in one copy
        pixels = d[base:]
        if self.augment is not None:
            params = d[2 * _DESC * n:base]
            self.be.augment2d(pixels, params, n, s["aug_max_hw"], s["aug_stages"], self._d_aug,
                              msrc=pixels if s["has_labels"] else None, mout=self._d_aug if s["has_labels"] else None,
                              ws=self._aug_ws)
            pixels = self._d_aug
        self.be.resize_linear(pixels, d[:_DESC * n].view(torch.int64).view(n, 2), s["d_img"])
        self.be.stage_images_u8(s["d_img"], s["x"])
        if s["has_labels"]:
            self.be.resize_linear(pixels, d[_DESC * n:2 * _DESC * n].view(torch.int64).view(n, 2), s["d_lab"])
            self.be.stage_labels_u8(s["d_lab"], s["y"], self.binarize)

    def get(self) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """The oldest queued batch: (x [N, 1, *spatial], y [N, *spatial] int64 or None).  The tensors belong to the slot:
        they are valid until ``slots`` further batches have been queued."""
        if self._got >= self._put:
            raise RuntimeError("InputStager: no batch queued")
        s = self._slots[self._got % len(self._slots)]
        self._got += 1
        if self._stream is not None:
            cur = torch.cuda.current_stream(self.device)
            cur.wait_event(s["ready"])
            ev = torch.cuda.Event()
            s["free"] = ev
            ev.record(cur)                     # refined by release(); until then: "whatever was queued before get()"
        return s["x"], (s["y"] if s["has_labels"] else None)

    def release(self) -> None:
        """Mark the batch taken by the last ``get()`` as consumed by everything queued on the current stream so far
        (call after the step's launches; ``put`` waits on it before overwriting that slot)."""
        s = self._slots[(self._got - 1) % len(self._slots)]
        if s.get("free") is not None:
            s["free"].record(torch.cuda.current_stream(self.device))


def stage_batch(images_u8: torch.Tensor, labels_u8: Optional[torch.Tensor] = None, dtype: torch.dtype = torch.float32,
                binarize_labels: bool = True, backend=None):
    """One-shot form on tensors that are already on the device: -> (x [N, 1, ...], y int64 or None)."""
    be = backend if backend is not None else runtime.get_backend(images_u8)
    x = torch.empty((images_u8.shape[0], 1) + tuple(images_u8.shape[1:]), dtype=dtype, device=images_u8.device)
    be.stage_images_u8(images_u8.contiguous(), x)
    y = None
    if labels_u8 is not None:
        y = torch.empty(labels_u8.shape, dtype=torch.int64, device=labels_u8.device)
        be.stage_labels_u8(labels_u8.contiguous(), y, binarize_labels)
    return x, y
