"""NetVLAD with fewer than 64 clusters on the CPU oracle: oracle/ibl_oracle.py reproduces the unmodified reference's
descriptors for K in {1, 8, 32, 48, 63} at two sizes and an EmbedNetPCA layer of input K*512
(tests/golden/clusters.npz, oracle/gen_golden_clusters.py)."""
import pytest
import torch

from conftest import load_golden, rel_l2
from oracle import ibl_oracle as O
from openibl_b200 import synth

KS = (1, 8, 32, 48, 63)
SIZES = (("s", 2, 64, 96, 21), ("l", 1, 240, 320, 22))   # oracle/gen_golden_clusters.py
SEED, PCA_K, PCA_DIM = 17, 32, 128


def _sd(K, with_pca=False):
    return synth.make_state_dict(seed=SEED, sharp=True, with_pca=with_pca, pca_dim=PCA_DIM, bias_scale=0.05,
                                 num_clusters=K)


@pytest.mark.parametrize("tag,b,h,w,img_seed", SIZES, ids=[s[0] for s in SIZES])
def test_oracle_raw_and_embednet_descriptors_for_every_cluster_count(tag, b, h, w, img_seed):
    g = load_golden("clusters")
    x = synth.make_images(seed=img_seed, batch=b, height=h, width=w)
    with torch.no_grad():
        feat = O.vgg16_trunk(x, _sd(KS[0]))           # the trunk's parameters do not depend on K
        for K in KS:
            sd = _sd(K)
            raw = O.netvlad(feat, sd["net_vlad.conv.weight"], sd["net_vlad.centroids"])
            assert raw.shape == (b, K, 512)
            assert rel_l2(raw[:, :, ::8], g[f"{tag}_k{K}_raw"]) < 1e-5, K
            assert rel_l2(O.vlad_normalize(raw)[:, ::4], g[f"{tag}_k{K}_vlad"]) < 1e-5, K


def test_oracle_embednetpca_with_pca_input_of_k_times_512():
    g = load_golden("clusters")
    _, b, h, w, img_seed = SIZES[0]
    sd = _sd(PCA_K, with_pca=True)
    assert tuple(sd["pca_layer.weight"].shape) == (PCA_DIM, PCA_K * 512, 1, 1)
    x = synth.make_images(seed=img_seed, batch=b, height=h, width=w)
    with torch.no_grad():
        assert rel_l2(O.embednetpca_forward(x, sd), g[f"pca_k{PCA_K}_desc"]) < 1e-5


def test_make_state_dict_default_is_64_clusters():
    a = synth.make_state_dict(seed=3, sharp=True, with_pca=True, pca_dim=16)
    b = synth.make_state_dict(seed=3, sharp=True, with_pca=True, pca_dim=16, num_clusters=64)
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    assert tuple(a["net_vlad.centroids"].shape) == (64, 512) and a["pca_layer.weight"].shape[1] == 32768
