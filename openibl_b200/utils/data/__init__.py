"""Loader helpers mirrored from ibl/utils/data/__init__.py:8-42."""
from .preprocessor import Preprocessor  # noqa: F401
from . import sampler  # noqa: F401

_MEAN = [0.48501960784313836, 0.4579568627450961, 0.4076039215686255]
_STD = [0.00392156862745098] * 3


class IterLoader:
    def __init__(self, loader, length=None):
        self.loader, self.length, self.iter = loader, length, None

    def __len__(self):
        return self.length if self.length is not None else len(self.loader)

    def new_epoch(self):
        self.iter = iter(self.loader)

    def next(self):
        try:
            return next(self.iter)
        except Exception:
            self.iter = iter(self.loader)
            return next(self.iter)


def get_transformer_train(height, width, device_decode=False):
    """device_decode=True: `Preprocessor` yields the file's bytes with the ColorJitter parameters drawn for it, and the
    trainers' `_parse_data` runs this same transform on the GPU (gpu_jpeg.decode_tuples), bit for bit."""
    import torchvision.transforms as T
    jitter = T.ColorJitter(0.7, 0.7, 0.7, 0.5)
    if device_decode:
        from .gpu_jpeg import DeviceJitterDecode
        return DeviceJitterDecode(height, width, jitter)
    return T.Compose([jitter, T.Resize((height, width)), T.ToTensor(), T.Normalize(mean=_MEAN, std=_STD)])


def get_transformer_test(height, width, tokyo=False, device_decode=False):
    """device_decode=True: `Preprocessor` yields the file's bytes and `extract_cnn_feature` runs this same transform
    on the GPU (gpu_jpeg.decode_to_tensor), bit for bit."""
    if device_decode:
        from .gpu_jpeg import DeviceDecode
        return DeviceDecode(height, width, tokyo)
    import torchvision.transforms as T
    return T.Compose([T.Resize(max(height, width) if tokyo else (height, width)), T.ToTensor(),
                      T.Normalize(mean=_MEAN, std=_STD)])
