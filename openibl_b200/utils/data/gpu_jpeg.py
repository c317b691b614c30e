"""The reference's test transform from JPEG file bytes, on the GPU (ibl/utils/data/__init__.py:37-42 after
ibl/utils/data/preprocessor.py:31-42: `Image.open(f).convert('RGB')`, `T.Resize`, `T.ToTensor`, `T.Normalize`).

A loader opts in with `get_transformer_test(h, w, tokyo, device_decode=True)`: `Preprocessor` then yields each file's
bytes as an `EncodedImage` (about 0.1 MB for a 480x640 JPEG instead of 3.7 MB of fp32), and `extract_cnn_feature`
turns a batch of them into the normalised fp32 tensor with `decode_to_tensor`:
  * `Engine.decode_jpeg_async` decodes baseline and progressive JPEGs (csrc/jpeg.cu) and 8-bit non-interlaced PNGs
    of every colour type (csrc/png.cu) on the device, bit-identical to Pillow;
  * files the device decoders do not take (CMYK, arithmetic-coded, progressive files libjpeg would block-smooth,
    16-bit or interlaced PNGs, ...) are decoded by Pillow on the host and join the same uint8 pipeline;
  * the existing Pillow-exact resize (`Engine.resize_u8`, skipped when the size already matches) and
    ToTensor + Normalize (`Engine.preprocess_u8`) finish the transform.
The result equals `get_transformer_test(h, w, tokyo)(Image.open(f).convert('RGB'))` bit for bit.

Training loaders opt in the same way with `get_transformer_train(h, w, device_decode=True)`: the worker draws the
`ColorJitter` parameters exactly as the host transform does and ships them with the bytes (`JitteredImage`); the
device applies the jitter (`Engine.color_jitter_u8`, csrc/color_jitter.cu) after the decode and before the resize, which
is the host transform's ColorJitter -> Resize order, and `decode_tuples` turns a collated tuple batch into the
trainers' [B, N, 3, H, W] input.  The result equals `get_transformer_train(h, w)(Image.open(f).convert('RGB'))` bit for
bit under the same torch RNG state."""
from __future__ import annotations

import io
from typing import List, Optional, Sequence

import numpy as np
import torch


class EncodedImage(bytes):
    """A file's bytes plus the output-size rule of the transform that will run on the device.  Being `bytes`, a
    batch of them passes torch's default collate (as a list) and `pin_memory` unchanged, and pickles to workers."""

    def __new__(cls, data: bytes, height: int, width: int, tokyo: bool = False, name: str = ""):
        obj = super().__new__(cls, data)
        obj.height, obj.width, obj.tokyo, obj.name = int(height), int(width), bool(tokyo), name
        return obj

    def __reduce__(self):
        return (EncodedImage, (bytes(self), self.height, self.width, self.tokyo, self.name))


class DeviceDecode:
    """Transform of `get_transformer_test(..., device_decode=True)`: wraps a file's bytes for the device pipeline."""

    def __init__(self, height: int, width: int, tokyo: bool = False):
        self.height, self.width, self.tokyo = int(height), int(width), bool(tokyo)

    def __call__(self, data: bytes, name: str = "") -> EncodedImage:
        return EncodedImage(data, self.height, self.width, self.tokyo, name)

    def __repr__(self):
        return f"DeviceDecode(height={self.height}, width={self.width}, tokyo={self.tokyo})"


class JitteredImage(EncodedImage):
    """An EncodedImage plus the `ColorJitter` parameters drawn for it: (order, brightness, contrast, saturation, hue)
    as `ColorJitter.get_params` returns them (order a list of 4 ints, None for a factor that is off)."""

    def __new__(cls, data: bytes, height: int, width: int, jitter, name: str = ""):
        obj = super().__new__(cls, data, height, width, False, name)
        order, *factors = jitter
        obj.jitter = (tuple(int(i) for i in order),) + tuple(None if v is None else float(v) for v in factors)
        return obj

    def __reduce__(self):
        return (JitteredImage, (bytes(self), self.height, self.width, self.jitter, self.name))


class DeviceJitterDecode(DeviceDecode):
    """Transform of `get_transformer_train(..., device_decode=True)`: draws the parameters of `color_jitter` (a
    `T.ColorJitter`) through `ColorJitter.get_params`, consuming the torch RNG exactly as the host transform does, and
    wraps them with the file's bytes.  The output size is `T.Resize((height, width))`'s."""

    def __init__(self, height: int, width: int, color_jitter):
        super().__init__(height, width, tokyo=False)
        self.color_jitter = color_jitter

    def __call__(self, data: bytes, name: str = "") -> JitteredImage:
        cj = self.color_jitter
        fn_idx, b, c, s, h = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
        return JitteredImage(data, self.height, self.width, (fn_idx.tolist(), b, c, s, h), name)

    def __repr__(self):
        return f"DeviceJitterDecode(height={self.height}, width={self.width}, color_jitter={self.color_jitter!r})"


def output_size(src_h: int, src_w: int, height: int, width: int, tokyo: bool = False):
    """(out_h, out_w) of `T.Resize(max(height, width) if tokyo else (height, width))` on a src_h x src_w PIL image
    (torchvision's _compute_resized_output_size for an int size: the short side becomes `size`, the long side
    int(size * long / short))."""
    if not tokyo:
        return int(height), int(width)
    size = max(height, width)
    short, long = (src_w, src_h) if src_w <= src_h else (src_h, src_w)
    new_short, new_long = size, int(size * long / short)
    return (new_long, new_short) if src_w <= src_h else (new_short, new_long)


def _host_decode(data: bytes) -> np.ndarray:
    from PIL import Image
    return np.array(Image.open(io.BytesIO(data)).convert("RGB"))


def decode_to_tensor(files: Sequence[bytes], height: int, width: int, tokyo: bool = False, device=None,
                     names: Optional[Sequence[str]] = None, pending: Optional[list] = None,
                     jitter: Optional[Sequence] = None) -> torch.Tensor:
    """JPEG or PNG file bytes -> fp32 [N,3,H,W] on the device, equal to the reference's test transform of the decoded image,
    or with `jitter` (one `ColorJitter.get_params` result per file) to its training transform.

    Corrupt entropy or zlib data is reported by the device after the fact: with `pending` None this call waits for
    the stream and raises RuntimeError naming the file; otherwise it appends (error words, names, PNG flags) to
    `pending` for `check_decode_errors` and does not synchronise."""
    from ... import _cabi
    from ...engine import Engine
    from . import _MEAN, _STD
    if len(files) == 0:
        raise ValueError("empty batch")
    eng = Engine.get(device)
    dev = torch.device("cuda", eng.device)
    names = list(names) if names is not None else [getattr(f, "name", "") or f"#{i}" for i, f in enumerate(files)]
    imgs, err = eng.decode_jpeg_async(files, fallback=_host_decode)     # rejected files: Pillow, same buffer
    if jitter is not None:
        eng.color_jitter_u8(imgs, jitter)              # ColorJitter at the source size, before Resize
    sizes = [output_size(im.shape[0], im.shape[1], height, width, tokyo) for im in imgs]
    if len(set(sizes)) != 1:
        raise ValueError(f"images of one batch resize to different sizes {sorted(set(sizes))}; "
                         "the reference's Tokyo loaders use batch size 1")
    oh, ow = sizes[0]
    u8 = torch.empty(len(imgs), oh, ow, 3, dtype=torch.uint8, device=dev)
    groups = {}
    for i, im in enumerate(imgs):
        groups.setdefault(tuple(im.shape[:2]), []).append(i)
    for (h, w), idx in groups.items():
        src = torch.stack([imgs[i] for i in idx])
        u8[idx] = src if (h, w) == (oh, ow) else eng.resize_u8(src, oh, ow)
    out = eng.preprocess_u8(u8, _MEAN, _STD)
    png = [bytes(f[:8]) == _cabi.PNG_SIGNATURE for f in files]
    if pending is None:
        check_decode_errors([(err, names, png)])
    else:
        pending.append((err, names, png))
    return out


def check_decode_errors(pending: List) -> None:
    """Raise RuntimeError naming the first file whose device decode reported corrupt entropy or zlib data."""
    for err, names, png in pending:
        bad = torch.nonzero(err).flatten().tolist()
        if bad:
            what = "corrupt PNG image data" if png[bad[0]] else "corrupt JPEG entropy data"
            raise RuntimeError(f"{what} in {names[bad[0]]!r}"
                               + (f" (and {len(bad) - 1} more in the batch)" if len(bad) > 1 else ""))
    pending.clear()


def is_encoded_batch(inputs) -> bool:
    return isinstance(inputs, (list, tuple)) and len(inputs) > 0 and all(isinstance(x, EncodedImage) for x in inputs)


def decode_batch(inputs: Sequence[EncodedImage], device=None, pending: Optional[list] = None) -> torch.Tensor:
    """A collated batch of EncodedImage -> the fp32 model input, with the size rule the carriers hold."""
    f0 = inputs[0]
    jittered = [isinstance(x, JitteredImage) for x in inputs]
    if any(jittered) and not all(jittered):
        raise ValueError("a batch mixes jittered training images with plain ones")
    return decode_to_tensor(inputs, f0.height, f0.width, f0.tokyo, device=device, names=[x.name for x in inputs],
                            pending=pending, jitter=[x.jitter for x in inputs] if all(jittered) else None)


def decode_tuples(inputs, device=None) -> torch.Tensor:
    """A collated training batch of tuples (the trainers' `_parse_data` input: inputs[n][0] holds the B carriers of
    tuple position n) -> fp32 [B, N, 3, H, W] on the device, all B*N images decoded in one call."""
    n, b = len(inputs), len(inputs[0][0])
    x = decode_batch([inputs[j][0][i] for i in range(b) for j in range(n)], device=device)
    return x.view(b, n, *x.shape[1:])
