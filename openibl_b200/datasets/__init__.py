"""Dataset registry (ibl/datasets/__init__.py:18-31): 'pitts' and 'tokyo' with the reference's constructor
signatures and attributes -- both arrange their json pair from the raw dbStruct .mat files on first use -- plus the
in-memory 'synthetic' split used by the parity tests and benchmarks, and `write_synthetic_pitts_tree` /
`write_synthetic_tokyo_tree` (Pittsburgh- and Tokyo-shaped trees of small images + dbStruct .mat files, for running
the reference's example scripts without the real data)."""
from .pitts import Pittsburgh
from .synthetic import SyntheticGallery, write_synthetic_pitts_tree, write_synthetic_tokyo_tree  # noqa: F401
from .tokyo import Tokyo

_factory = {"pitts": Pittsburgh, "tokyo": Tokyo, "synthetic": SyntheticGallery}


def names():
    return sorted(_factory.keys())


def create(name, root, *args, **kwargs):
    if name not in _factory:
        raise KeyError("Unknown dataset:", name)
    return _factory[name](root, *args, **kwargs)


def get_dataset(name, root, *args, **kwargs):
    import warnings
    warnings.warn("get_dataset is deprecated. Use create instead.")
    return create(name, root, *args, **kwargs)
