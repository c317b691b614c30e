"""Test harness ONLY: a minimal `h5py` stand-in that stores a "file" as an .npz archive, for running the unmodified
training recipe (examples/cluster.py, examples/netvlad_img.py), which really reads and writes HDF5 files.

Covers what those scripts and openibl_b200/pca.py use: `File(path, mode)` as a context manager, `create_dataset(name,
shape, dtype=...)` or `create_dataset(name, data=...)`, slice assignment into a dataset, `get(name)`, `f[name]`,
`dataset[...]`, `keys()`.  The archive is written to `path` itself (no extension added) when a writable file closes.
The empty stand-in in ../stubs/h5py stays as it is: the product switches on `hasattr(h5py, "File")`."""
import numpy as np


class Dataset:
    def __init__(self, array):
        self._a = array

    shape = property(lambda self: self._a.shape)
    dtype = property(lambda self: self._a.dtype)

    def __len__(self):
        return len(self._a)

    def __getitem__(self, index):
        return np.array(self._a[index])

    def __setitem__(self, index, value):
        self._a[index] = value

    def __array__(self, dtype=None, copy=None):
        return np.asarray(self._a, dtype=dtype)


class File:
    def __init__(self, name, mode="r"):
        self.filename, self.mode = str(name), mode
        self._writable = mode != "r"
        self._data = {}
        if mode in ("r", "r+", "a"):
            try:
                with np.load(self.filename) as z:
                    self._data = {k: Dataset(z[k].copy()) for k in z.files}
            except FileNotFoundError:
                if mode != "a":
                    raise

    def create_dataset(self, name, shape=None, dtype=None, data=None):
        if name in self._data:
            raise ValueError("dataset %r already exists" % name)
        if data is not None:
            arr = np.array(data, dtype=dtype)
        else:
            arr = np.zeros(tuple(shape), dtype=dtype or np.float32)
        self._data[name] = Dataset(arr)
        return self._data[name]

    def get(self, name, default=None):
        return self._data.get(name, default)

    def __getitem__(self, name):
        return self._data[name]

    def __contains__(self, name):
        return name in self._data

    def keys(self):
        return self._data.keys()

    def close(self):
        if self._writable:
            with open(self.filename, "wb") as f:
                np.savez(f, **{k: d._a for k, d in self._data.items()})
            self._writable = False

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False
