"""Synthetic place-recognition data.

SyntheticGallery: in-memory split with the reference dataset's attribute names (q_test / db_test / test_pos,
items = (fname, pid, x, y); ibl/utils/data/dataset.py) -- images are generated from seeds by the callers.

write_synthetic_pitts_tree: a Pittsburgh-shaped tree ON DISK -- NetVLAD-style dbStruct .mat files for the
train / val / test splits and small JPEG images laid out as `raw/Pittsburgh/{images,queries}/...` -- so that
code written for the real dataset (the reference's examples/test.py) runs end to end through
`datasets.create('pitts', root, scale='30k')`, PIL decoding and the torchvision transforms.

write_synthetic_tokyo_tree: the same for Tokyo -- Time Machine and Tokyo 24/7 dbStruct .mat files, JPEGs and the PNG
database -- shaped to exercise every rule of the Tokyo arrangement, for `datasets.create('tokyo', root)`."""
import os
import os.path as osp

import numpy as np


class SyntheticGallery:
    def __init__(self, root=None, n_db=1000, n_q=100, scale=None, verbose=False, seed=0):
        rng = np.random.RandomState(seed)
        self.images_dir = root
        self.db_test = [("db/%06d.jpg" % i, i, float(i), 0.0) for i in range(n_db)]
        pos = rng.randint(0, n_db, size=n_q)
        self.q_test = [("q/%06d.jpg" % i, n_db + i, float(pos[i]), 0.0) for i in range(n_q)]
        self.test_pos = [np.array([int(p)]) for p in pos]


def _scene(rng, h, w, street):
    """A smooth colour field shared by the whole `street` (places of one street look alike, as real ones do) plus
    a few rectangles of its own: compresses like a photo, similar to its neighbours, not identical."""
    img = street.copy()
    for _ in range(3):
        y0, x0 = rng.randint(0, h - 8), rng.randint(0, w - 8)
        y1, x1 = y0 + rng.randint(6, h // 3), x0 + rng.randint(6, w // 3)
        img[y0:y1, x0:x1] = rng.randint(0, 256, size=3)
    return img


def _street(rng, h, w):
    from PIL import Image
    coarse = rng.randint(0, 256, size=(6, 8, 3)).astype(np.uint8)
    return np.asarray(Image.fromarray(coarse).resize((w, h), Image.BICUBIC)).astype(np.int16)


def write_synthetic_pitts_tree(root, scale="30k", n_places=(24, 10, 40), views=2, size=(120, 160), seed=0):
    """Writes <root>/raw/pitts<scale>_{train,val,test}.mat and the JPEGs they name.

    Each split has n database places on a 100 m grid with `views` images each and one query place 4 m from
    every second database place (its image is a perturbed view of that place), so every query has exactly one
    positive place inside the 10 m / 25 m radii the reference uses (dataset.py:103-110).  Returns the root."""
    from PIL import Image
    from scipy.io import savemat
    rng = np.random.RandomState(seed)
    raw = osp.join(root, "raw")
    h, w = size
    pano = 0
    for split, n_db in zip(("train", "val", "test"), n_places):
        db_names, db_utm, q_names, q_utm = [], [], [], []
        for p in range(n_db):
            if p % 8 == 0:
                street = _street(rng, h, w)
            scene = _scene(rng, h, w, street)
            x, y = 1000.0 * (("train", "val", "test").index(split) + 1) + 100.0 * (p % 6), 100.0 * (p // 6)
            sid = "%06d" % pano
            pano += 1
            for v in range(views):
                name = osp.join("%03d" % (pano // 1000), "%s_pitch%d_yaw%d.jpg" % (sid, 1, v + 1))
                view = np.clip(np.roll(scene, 3 * v, axis=1) + rng.randint(-6, 7, size=scene.shape), 0, 255)
                _save(Image, osp.join(raw, "Pittsburgh", "images", name), view)
                db_names.append(name)
                db_utm.append((x, y))
            if p % 2 == 0:
                qsid = "%06d" % pano
                pano += 1
                name = osp.join("%03d" % (pano // 1000), "%s_pitch1_yaw1.jpg" % qsid)
                view = np.clip(np.roll(scene, -6, axis=1) + rng.randint(-40, 41, size=scene.shape), 0, 255)
                _save(Image, osp.join(raw, "Pittsburgh", "queries", name), view)
                q_names.append(name)
                q_utm.append((x + 4.0, y))
        cell = lambda names: np.array([[n] for n in names], dtype=object)
        st = {"whichSet": split, "dbImageFns": cell(db_names), "utmDb": np.asarray(db_utm, dtype=np.float64).T,
              "qImageFns": cell(q_names), "utmQ": np.asarray(q_utm, dtype=np.float64).T,
              "numImages": float(len(db_names)), "numQueries": float(len(q_names))}
        os.makedirs(raw, exist_ok=True)
        savemat(osp.join(raw, "pitts%s_%s.mat" % (scale, split)), {"dbStruct": st})
    return root


def write_synthetic_tokyo_tree(root, n_places=(12, 9, 8), views=2, size=(120, 160), seed=0):
    """Writes <root>/raw/tokyoTM_{train,val}.mat, <root>/raw/tokyo247.mat and the images they name, laid out as the
    Tokyo loader reads them: `raw/tokyoTM/images/<group>/<place>/<time stamp>/<file>.jpg`,
    `raw/tokyo247/query/<file>.jpg` and `raw/tokyo247/images/<place>/<file>.png` (named .jpg in the struct).

    Time Machine: place p of a split has 1 + p % 3 time stamps of `views` images each; the first view of every time
    stamp is listed as a query image, the others as database images, and one path is listed twice.  Places come in
    pairs 4 m apart on a 100 m grid, both views of one scene, so every identity has a positive within 10 m.
    Tokyo 24/7: n places of `views` database images; every place gets a query 4 m away, two for every third place
    (at the same UTM position, so they form one query place), landscape and portrait at four sizes.  Returns the root."""
    from PIL import Image
    from scipy.io import savemat
    rng = np.random.RandomState(seed)
    raw = osp.join(root, "raw")
    h, w = size
    cell = lambda names: np.array([[n] for n in names], dtype=object)
    utm_of = lambda pts: np.asarray(pts, dtype=np.float64).reshape(-1, 2).T
    n_place = 0
    for split, n in zip(("train", "val"), n_places[:2]):
        q_names, q_utm, db_names, db_utm = [], [], [], []
        for p in range(n):
            if p % 2 == 0:
                scene = _scene(rng, h, w, _street(rng, h, w))
            x = 360000.5 + 1000.0 * ("train", "val").index(split) + 100.0 * (p // 2 % 6) + 4.0 * (p % 2)
            y = 3940000.25 + 100.0 * (p // 12)
            place = "%05d" % n_place
            n_place += 1
            stamps = ["%d%02d" % (2009 + t, 1 + 5 * t) for t in range(1 + p % 3)]
            for t, ts in enumerate(stamps if p % 2 == 0 else stamps[::-1]):      # first-seen order != name order
                light = 18 * t - 12
                for v in range(views):
                    name = "%02d/%s/%s/%s_%s_v%d.jpg" % (n_place // 50, place, ts, place, ts, v)
                    view = np.clip(np.roll(scene, 3 * v + 5 * (p % 2), axis=1) + light
                                   + rng.randint(-6, 7, size=scene.shape), 0, 255)
                    _save(Image, osp.join(raw, "tokyoTM", "images", name), view)
                    (q_names if v == 0 else db_names).append(name)
                    (q_utm if v == 0 else db_utm).append((x, y))
        db_names.append(q_names[0])                      # listed twice: registered once
        db_utm.append(q_utm[0])
        st = {"whichSet": split, "dbImageFns": cell(db_names), "utmDb": utm_of(db_utm),
              "dbTimeStamp": np.arange(len(db_names), dtype=np.float64)[None],
              "qImageFns": cell(q_names), "utmQ": utm_of(q_utm),
              "qTimeStamp": np.arange(len(q_names), dtype=np.float64)[None],
              "numImages": float(len(db_names)), "numQueries": float(len(q_names))}
        os.makedirs(raw, exist_ok=True)
        savemat(osp.join(raw, "tokyoTM_%s.mat" % split), {"dbStruct": st})

    q_sizes = ((h, w), (w, h), (h * 4 // 5, w * 9 // 10), (w * 9 // 10, h * 4 // 5))   # landscape / portrait
    q_names, q_utm, db_names, db_utm = [], [], [], []
    n_q = 0
    for p in range(n_places[2]):
        if p % 8 == 0:
            street = _street(rng, h, w)
        scene = _scene(rng, h, w, street)
        x, y = 381234.567 + 100.0 * (p % 6), 3946789.125 + 100.0 * (p // 6)
        for v in range(views):
            name = "%05d/%05d%03d.jpg" % (p, p, v)
            view = np.clip(np.roll(scene, 3 * v, axis=1) + rng.randint(-6, 7, size=scene.shape), 0, 255)
            _save(Image, osp.join(raw, "tokyo247", "images", name[:-3] + "png"), view)
            db_names.append(name)
            db_utm.append((x, y))
        for _ in range(2 if p % 3 == 0 else 1):
            qh, qw = q_sizes[n_q % len(q_sizes)]
            view = np.clip(np.roll(scene, -6 - 2 * n_q, axis=1) + rng.randint(-40, 41, size=scene.shape), 0, 255)
            view = np.asarray(Image.fromarray(view.astype(np.uint8)).resize((qw, qh), Image.BILINEAR))
            name = "%06d.jpg" % (100 * p + n_q)
            _save(Image, osp.join(raw, "tokyo247", "query", name), view)
            q_names.append(name)
            q_utm.append((x + 4.0, y))
            n_q += 1
    st = {"whichSet": "test", "dbImageFns": cell(db_names), "utmDb": utm_of(db_utm),
          "qImageFns": cell(q_names), "utmQ": utm_of(q_utm),
          "numImages": float(len(db_names)), "numQueries": float(len(q_names))}
    savemat(osp.join(raw, "tokyo247.mat"), {"dbStruct": st})
    return root


def _save(Image, path, arr):
    os.makedirs(osp.dirname(path), exist_ok=True)
    Image.fromarray(arr.astype(np.uint8)).save(path, quality=92)
