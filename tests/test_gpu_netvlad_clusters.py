"""NetVLAD layers of 1..64 clusters (`models.create('netvlad', num_clusters=K)`) through extraction, training and
retrieval, against the unmodified reference run on CPU (tests/golden/clusters.npz, oracle/gen_golden_clusters.py) and
the CPU oracle.  The tensor-core kernel pads K < 64 clusters to 64; the CUDA-core kernels mask the clusters past K.
Tolerances: the north-star 1e-4 relative L2 for descriptors, and those of test_gpu_trainer.py / test_gpu_train.py for
the training steps (stated there)."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden, rel_l2
from openibl_b200 import synth

pytestmark = pytest.mark.gpu

DESC_TOL = 1e-4
KS = (1, 8, 32, 48, 63)
SIZES = (("s", 2, 64, 96, 21), ("l", 1, 240, 320, 22))   # oracle/gen_golden_clusters.py
SEED, PCA_K, PCA_DIM = 17, 32, 128
# (name, conv mode, gemm mode): the fused tensor-core path, and fp32 CUDA cores throughout
MODES = (("tc", 1, 1), ("simt", 0, 0))


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    e = Engine.get(0)
    yield e
    e.conv_mode = 1
    e.set_gemm_mode(1)


@pytest.fixture(scope="module")
def golden():
    return load_golden("clusters")


@pytest.fixture(scope="module")
def oracle_feat():
    """Reference-order conv5_3 maps of the two golden sizes on the CPU (the trunk does not depend on K)."""
    from oracle import ibl_oracle as O
    sd = _sd(KS[0])
    with torch.no_grad():
        return {tag: O.vgg16_trunk(synth.make_images(seed=s, batch=b, height=h, width=w), sd)
                for tag, b, h, w, s in SIZES}


def _sd(K, seed=SEED, bias_scale=0.05, with_pca=True):
    return synth.make_state_dict(seed=seed, sharp=True, with_pca=with_pca, pca_dim=PCA_DIM, bias_scale=bias_scale,
                                 num_clusters=K)


def _models(K):
    from ibl import models
    base = models.create("vgg16", pretrained=False)
    nv = models.create("netvlad", num_clusters=K, dim=512)
    pca = models.create("embednetpca", base, nv, dim=PCA_DIM)
    pca.load_state_dict(_sd(K))
    pca = pca.cuda().eval()
    return models.create("embednet", pca.base_model, pca.net_vlad).cuda().eval(), pca


@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("tag,b,h,w,img_seed", SIZES, ids=[s[0] for s in SIZES])
def test_embednet_and_pca_descriptors_both_modes(eng, golden, oracle_feat, K, tag, b, h, w, img_seed):
    """EmbedNet against the reference golden, EmbedNetPCA (PCA input K*512) against the oracle on the reference's
    feature map and the golden at K = 32, in both math modes."""
    from oracle import ibl_oracle as O
    sd = _sd(K)
    with torch.no_grad():
        v = O.vlad_normalize(O.netvlad(oracle_feat[tag], sd["net_vlad.conv.weight"], sd["net_vlad.centroids"]))
        want_pca = O.pca_whiten(v, sd["pca_layer.weight"], sd["pca_layer.bias"])
    emb, embpca = _models(K)
    x = synth.make_images(seed=img_seed, batch=b, height=h, width=w).cuda()
    for name, conv, gemm in MODES:
        eng.conv_mode = conv
        eng.set_gemm_mode(gemm)
        with torch.no_grad():
            _, vlad = emb(x)
            desc = embpca(x)
        assert tuple(vlad.shape) == (b, K * 512) and tuple(desc.shape) == (b, PCA_DIM)
        assert rel_l2(vlad[:, ::4].cpu(), golden[f"{tag}_k{K}_vlad"]) < DESC_TOL, (name, rel_l2(vlad[:, ::4].cpu(), golden[f"{tag}_k{K}_vlad"]))
        assert rel_l2(desc.cpu(), want_pca) < DESC_TOL, (name, rel_l2(desc.cpu(), want_pca))
        if K == PCA_K and tag == "s":
            assert rel_l2(desc.cpu(), golden[f"pca_k{K}_desc"]) < DESC_TOL, name


@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("tag,b,h,w,img_seed", SIZES, ids=[s[0] for s in SIZES])
def test_netvlad_forward_raw_nhwc_tensor_cores_and_nchw_cuda_cores(eng, golden, K, tag, b, h, w, img_seed):
    """NetVLAD.forward's raw [N,K,512] output: the nchw CUDA-core branch (what the module calls) and the nhwc
    tensor-core branch, on the fp32 trunk's feature map."""
    emb, _ = _models(K)
    eng.conv_mode = 0
    x = synth.make_images(seed=img_seed, batch=b, height=h, width=w).cuda()
    want = golden[f"{tag}_k{K}_raw"]
    with torch.no_grad():
        _, feat = emb.base_model(x)
        raw = emb.net_vlad(feat)
        assert tuple(raw.shape) == (b, K, 512)
        assert rel_l2(raw[:, :, ::8].cpu(), want) < DESC_TOL, rel_l2(raw[:, :, ::8].cpu(), want)
        eng.set_gemm_mode(1)
        raw_tc, _ = eng.netvlad_forward(feat.permute(0, 2, 3, 1).contiguous(), emb.net_vlad.conv.weight,
                                        emb.net_vlad.centroids, nhwc=True, want_raw=True, want_norm=False)
        assert tuple(raw_tc.shape) == (b, K, 512)
        assert rel_l2(raw_tc[:, :, ::8].cpu(), want) < DESC_TOL, rel_l2(raw_tc[:, :, ::8].cpu(), want)
    eng.conv_mode = 1


def _guarded(n_valid, sentinel=-12345.0, guard=4096):
    buf = torch.full((n_valid + guard,), sentinel, device="cuda")
    return buf, buf[:n_valid], buf[n_valid:]


@pytest.mark.parametrize("K", [1, 48])
def test_outputs_followed_by_a_guard_region_stay_in_bounds(eng, K):
    """The last image's rows end exactly where the caller's buffer ends; a sentinel-filled guard behind it must be
    untouched by every path: fused extraction, and NetVLAD forward through the nhwc tensor-core and the nchw / nhwc
    CUDA-core kernels (raw and normalised outputs)."""
    from openibl_b200.engine import OUT_VLAD, _ptr, _stream
    from oracle import ibl_oracle as O
    emb, _ = _models(K)
    N, H, W = 3, 240, 320                       # 300 feature pixels: three tiles, three units per image
    x = synth.make_images(seed=5, batch=N, height=H, width=W).cuda()
    D = K * 512
    eng.conv_mode = 1
    eng.set_gemm_mode(1)
    with torch.no_grad():
        _, want = emb(x)
        buf, out, tail = _guarded(N * D)
        ok = eng.lib.ibl_extract(eng.h, _ptr(x), N, H, W, OUT_VLAD, _ptr(out), _ptr(None), _stream(eng.device))
        torch.cuda.synchronize()
        assert ok == 0 and bool((tail == -12345.0).all()), "fused extraction wrote past its output"
        assert torch.equal(out.view(N, D), want)
        eng.conv_mode = 0
        _, feat = emb.base_model(x)
        eng.conv_mode = 1
        sd = {k: v.cpu() for k, v in emb.net_vlad.state_dict().items()}
        ref = O.netvlad(feat.cpu(), sd["conv.weight"], sd["centroids"])
        w, c = emb.net_vlad.conv.weight.detach().reshape(K, 512), emb.net_vlad.centroids.detach()
        S = feat.shape[2] * feat.shape[3]
        for nhwc, gemm in ((1, 1), (1, 0), (0, 0)):
            eng.set_gemm_mode(gemm)
            f = feat.permute(0, 2, 3, 1).contiguous() if nhwc else feat.contiguous()
            rbuf, raw, rtail = _guarded(N * D)
            nbuf, nrm, ntail = _guarded(N * D)
            ok = eng.lib.ibl_netvlad_forward(eng.h, _ptr(f), nhwc, N, 512, S, _ptr(w), _ptr(c), K, 1, _ptr(raw),
                                             _ptr(nrm), _stream(eng.device))
            torch.cuda.synchronize()
            assert ok == 0
            assert bool((rtail == -12345.0).all()) and bool((ntail == -12345.0).all()), (nhwc, gemm)
            assert rel_l2(raw.view(N, K, 512).cpu(), ref) < DESC_TOL, (nhwc, gemm)
            assert rel_l2(nrm.view(N, D).cpu(), O.vlad_normalize(ref)) < DESC_TOL, (nhwc, gemm)
    eng.set_gemm_mode(1)


def _freeze_below_conv5(trunk):
    for layer in list(trunk.base.children())[:24]:
        for p in layer.parameters():
            p.requires_grad = False


def test_trainer_triplet_step_k32_vs_reference_golden(eng, golden):
    """Trainer._forward, triplet loss on EmbedNet's VLAD with 32 clusters (tolerances of test_gpu_trainer.py)."""
    from ibl import models
    from ibl.trainers import Trainer
    K = 32
    m = models.create("embednet", models.create("vgg16", pretrained=False), models.create("netvlad", num_clusters=K,
                                                                                          dim=512))
    m.load_state_dict(_sd(K, seed=13, bias_scale=0.02, with_pca=False))
    _freeze_below_conv5(m.base_model)
    m = m.cuda().train()
    easy, _ = synth.make_sfrs_tuples(seed=41, tuples=2, neg_num=3, n_diff=1, height=64, width=96)
    loss = Trainer(m, margin=0.1 ** 0.5, gpu=0)._forward(easy.cuda(), True, "triplet")
    want = float(golden["train_loss"])
    assert abs(loss.item() - want) < 2e-4 * max(1.0, abs(want)), (loss.item(), want)
    loss.backward()
    base = m.base_model.base
    for slot in (24, 26, 28):
        gw = base[slot].weight.grad.cpu()
        sub, ref = gw[::16, ::8].double().flatten(), torch.from_numpy(golden[f"train_w{slot}"]).double().flatten()
        assert rel_l2(sub, ref) < 2e-2, (slot, rel_l2(sub, ref))
        assert float(sub @ ref / (sub.norm() * ref.norm())) > 0.9998, slot
        wnorm = float(golden[f"train_w{slot}_norm"])
        assert abs(float(gw.double().norm()) - wnorm) < 1e-2 * wnorm
        assert rel_l2(base[slot].bias.grad.cpu(), golden[f"train_b{slot}"]) < 2e-2, slot
    cg, wg = m.net_vlad.centroids.grad, m.net_vlad.conv.weight.grad
    assert tuple(cg.shape) == (K, 512) and tuple(wg.shape[:2]) == (K, 512) and wg[0].numel() == 512
    assert rel_l2(cg.cpu()[:, ::4], golden["train_centroids"]) < 3e-3
    assert rel_l2(wg.cpu()[:, ::4, 0, 0], golden["train_conv_w"]) < 3e-3


def test_sfrs_region_step_k16_vs_reference_golden(eng, golden):
    """SFRSTrainer._forward generation 1 (hard-region + soft loss) on EmbedRegionNet with 16 clusters, tuple_size 2
    (the reference's result is the mean of two single-tuple runs); tolerances of the SFRS step test."""
    from ibl import models
    from ibl.trainers import SFRSTrainer
    K, B, NEG = 16, 2, 2

    def build(seed):
        m = models.create("embedregionnet", models.create("vgg16", pretrained=False),
                          models.create("netvlad", num_clusters=K, dim=512), tuple_size=B)
        m.load_state_dict(_sd(K, seed=seed, bias_scale=0.02, with_pca=False))
        _freeze_below_conv5(m.base_model)
        return m.cuda().train()

    easy, diff = synth.make_sfrs_tuples(seed=31, tuples=B, neg_num=NEG, n_diff=2, height=64, width=96)
    model, cache = build(13), build(23)
    tr = SFRSTrainer(model, cache, margin=0.1, neg_num=NEG, gpu=0, temp=[0.07, 0.07])
    lh, ls = tr._forward(easy.cuda(), diff.cuda(), "sare_ind", 1)
    for got, key in ((lh, "sfrs_loss_hard"), (ls, "sfrs_loss_soft")):
        want = float(golden[key])
        assert abs(got.item() - want) < 2e-4 * max(1.0, abs(want)), (key, got.item(), want)
    (lh + 0.5 * ls).backward()
    base = model.base_model.base
    for slot in (24, 26, 28):
        gw = base[slot].weight.grad.cpu()
        sub, want = gw[::8, ::8].double().flatten(), torch.from_numpy(golden[f"sfrs_w{slot}"]).double().flatten()
        assert rel_l2(sub, want) < 2e-2, (slot, rel_l2(sub, want))
        assert float(sub @ want / (sub.norm() * want.norm())) > 0.9998, slot
        wnorm = float(golden[f"sfrs_w{slot}_norm"])
        assert abs(float(gw.double().norm()) - wnorm) < 1e-2 * wnorm
        assert rel_l2(base[slot].bias.grad.cpu(), golden[f"sfrs_b{slot}"]) < 2e-2, slot
    assert tuple(model.net_vlad.centroids.grad.shape) == (K, 512)
    assert rel_l2(model.net_vlad.centroids.grad.cpu()[:, ::4], golden["sfrs_centroids"]) < 3e-3
    assert rel_l2(model.net_vlad.conv.weight.grad.cpu()[:, ::4, 0, 0], golden["sfrs_conv_w"]) < 3e-3


def test_gallery_extraction_pca_and_evaluator_k32_match_oracle_recalls(eng, tmp_path):
    """A synthetic gallery end to end at K = 32: EmbedNet extraction (16,384-d raw descriptors), PCA fit on them,
    Evaluator.evaluate with PCA, with and without re-ranking.  The recalls equal the CPU oracle's on the same
    descriptors' distances."""
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    from eval_synthetic import SeededImages
    from torch.utils.data import DataLoader
    from ibl import datasets, models
    from ibl.evaluators import Evaluator, extract_features
    from ibl.pca import PCA
    from ibl.utils.data.sampler import DistributedSliceSampler
    from oracle import ibl_oracle as O
    from openibl_b200.utils.rerank import re_ranking
    K, H, W, P = 32, 64, 96, 24
    eng.conv_mode = 1
    eng.set_gemm_mode(1)
    ds = datasets.create("synthetic", None, n_db=40, n_q=12, seed=0)

    def loader(items):
        return DataLoader(SeededImages(items, H, W), batch_size=5, num_workers=0,
                          sampler=DistributedSliceSampler(items, num_replicas=1, rank=0), shuffle=False)

    torch.manual_seed(0)
    nv = models.create("netvlad", num_clusters=K, dim=512)
    p = synth.make_netvlad_params(seed=0, num_clusters=K, sharp=True)
    nv.centroids.data.copy_(p["centroids"])
    nv.conv.weight.data.copy_(p["conv_weight"])
    model = models.create("embednet", models.create("vgg16", pretrained=False), nv).cuda()
    dataset = sorted(set(ds.q_test) | set(ds.db_test))
    raw = extract_features(model, loader(dataset), dataset, vlad=True)
    assert next(iter(raw.values())).shape == (K * 512,)
    pca = PCA(P, True, str(tmp_path / "pca.h5"))
    pca.train(torch.stack([raw[f] for f, _, _, _ in ds.db_test]).cuda())
    feats = extract_features(model, loader(dataset), dataset, vlad=True, pca=pca)
    q = torch.stack([feats[f] for f, _, _, _ in ds.q_test])
    db = torch.stack([feats[f] for f, _, _, _ in ds.db_test])
    assert q.shape == (12, P)
    pids = [x[1] for x in ds.db_test]
    d = O.pairwise_distance(q, db).numpy()
    want = O.evaluate_all(d, ds.test_pos, pids)
    ev = Evaluator(model)
    got = ev.evaluate(loader(ds.q_test), dataset, ds.q_test, ds.db_test, ds.test_pos, gallery_loader=loader(ds.db_test),
                      vlad=True, pca=pca)
    assert np.allclose(got, want, atol=1e-9), (got, want)
    d_rr = re_ranking(d, O.pairwise_distance(q, q).numpy(), O.pairwise_distance(db, db).numpy(), k1=10, k2=1,
                      lambda_value=0.3)
    want_rr = O.evaluate_all(d_rr, ds.test_pos, pids)
    got_rr = ev.evaluate(loader(ds.q_test), dataset, ds.q_test, ds.db_test, ds.test_pos,
                         gallery_loader=loader(ds.db_test), vlad=True, pca=pca, rerank=True, rr_topk=10,
                         lambda_value=0.3)
    assert np.allclose(got_rr, want_rr, atol=1e-9), (got_rr, want_rr)


@pytest.mark.parametrize("K,status", [(0, 1), (65, 6), (128, 6)])
def test_cluster_counts_outside_1_to_64_raise_naming_the_range(eng, K, status):
    from ibl import models
    from openibl_b200._cabi import IblError
    layer = models.create("netvlad", num_clusters=K, dim=512).cuda()
    x = torch.randn(1, 512, 4, 5, device="cuda")
    for grad in (False, True):
        with torch.set_grad_enabled(grad), pytest.raises(IblError, match=r"1\.\.64") as e:
            layer(x)
        assert e.value.status == status
