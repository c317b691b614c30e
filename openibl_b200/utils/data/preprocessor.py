"""Image list -> (img, fname, pid, x, y) samples (ibl/utils/data/preprocessor.py:15-42)."""
import os.path as osp

from torch.utils.data import Dataset

from .gpu_jpeg import DeviceDecode


class Preprocessor(Dataset):
    def __init__(self, dataset, root=None, transform=None):
        super().__init__()
        self.dataset, self.root, self.transform = dataset, root, transform

    def __len__(self):
        return len(self.dataset)

    def __getitem__(self, indices):
        if isinstance(indices, (tuple, list)):
            return [self._one(i) for i in indices]
        return self._one(indices)

    def _one(self, index):
        from PIL import Image
        fname, pid, x, y = self.dataset[index]
        fpath = fname if self.root is None else osp.join(self.root, fname)
        if isinstance(self.transform, DeviceDecode):     # decode + transform (+ jitter) happen on the GPU (gpu_jpeg.py)
            with open(fpath, "rb") as f:
                return self.transform(f.read(), fname), fname, pid, x, y
        img = Image.open(fpath).convert("RGB")
        if self.transform is not None:
            img = self.transform(img)
        return img, fname, pid, x, y
