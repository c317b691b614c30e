"""Host-side mirror of the reference's model plugin API (ibl/models/__init__.py:7-53).

Same registry names, constructor signatures, attributes and state-dict keys as the reference
(SURVEY 8b), so checkpoints and `examples/test.py` work unchanged -- but `forward` does not run
torch ops: it hands raw device pointers to libiblb200.so.  Parameters stay ordinary
`nn.Parameter`s (DDP wrapping, `.cuda()`, `load_state_dict`, `copy_state_dict` all work);
the engine re-lays them out when their version counters change.

No CPU path: calling a model on CPU tensors raises.  Training (config 5, SURVEY 8 f1): NetVLAD and the trainable
suffix of the VGG trunk (conv5_x when `train_layers='conv5'`, vgg.py:50-53) are `torch.autograd.Function`s whose
forward AND backward run in libiblb200 (Hopper wgmma dgrad / wgrad, NetVLAD backward kernels); the region algebra of
EmbedRegionNet's train branch (sums of quarter VLADs, two normalisations, a 9x9 matmul per pair) stays in torch.
EmbedNetPCA trains end to end: its PCA layer is a third such Function (tensor-core dgrad / wgrad in libiblb200).
"""
from __future__ import annotations

import torch
from torch import nn

from .engine import Engine, invalidate_caches
from .synth import VGG16_PLAN

__all__ = ["VGG", "vgg16", "NetVLAD", "EmbedNet", "EmbedNetPCA", "EmbedRegionNet", "create", "names"]


_POOL_AFTER = [i for i, item in enumerate(VGG16_PLAN) if item == "P"]


def _layer_table():
    """[(cin, cout, relu, pool)] for the 13 conv layers, in order."""
    convs, pools = [], set()
    for item in VGG16_PLAN:
        if item == "P":
            pools.add(len(convs) - 1)
        else:
            convs.append(item)
    return [(c[1], c[2], i != len(convs) - 1, i in pools) for i, c in enumerate(convs)]


class _VGGTrunkFunction(torch.autograd.Function):
    """VGG.forward with a trainable suffix (layers first..12): frozen prefix on the inference kernels, then one
    conv(+ReLU) at a time keeping (input, post-ReLU output) for the backward; pools are separate so that the pre-pool
    activation is available.  Backward: ReLU mask + tensor-core dgrad/wgrad per layer (ibl_vgg16_layer_backward),
    first-maximum 2x2 pool backward.  Gradients come back in the parameters' own layouts (OIHW, [Cout])."""

    @staticmethod
    def forward(ctx, x, first, *params):
        eng = Engine.get(x.device)
        table = _layer_table()
        a = eng.vgg16_prefix_forward(x, first) if first > 0 else x.contiguous()
        saved = []
        for l in range(first, 13):
            cin, cout, relu, pool = table[l]
            y = eng.vgg16_layer_forward(l, a, cout)
            saved.append(a)
            saved.append(y)
            a = eng.maxpool2x2(y) if pool else y
        ctx.first = first
        ctx.w_shapes = [tuple(p.shape) for p in params[0::2]]
        ctx.save_for_backward(*saved)
        return a.permute(0, 3, 1, 2).contiguous()            # the reference returns NCHW (vgg.py:70)

    @staticmethod
    def backward(ctx, grad_nchw):
        saved = ctx.saved_tensors
        eng = Engine.get(grad_nchw.device)
        table = _layer_table()
        first = ctx.first
        g = grad_nchw.permute(0, 2, 3, 1).contiguous()
        grads = [None] * (2 * (13 - first))
        for l in range(12, first - 1, -1):
            i = l - first
            a_in, y = saved[2 * i], saved[2 * i + 1]
            cin, cout, relu, pool = table[l]
            if pool:
                g = eng.maxpool2x2_backward(y, g)
            gx, gw, gb = eng.vgg16_layer_backward(l, a_in, y if relu else None, g, ctx.w_shapes[i], need_gx=l > first)
            grads[2 * i], grads[2 * i + 1] = gw, gb
            g = gx
        return (None, None, *grads)


class VGG(nn.Module):
    """Reference ibl/models/vgg.py:15-87.  `base` holds the 13 conv layers at the torchvision
    `features[:-2]` indices so the state-dict keys are base.{0,2,...,28}.{weight,bias}."""

    _fix_layers = {"conv5": 24, "conv4": 17, "conv3": 10, "conv2": 5, "full": 0}

    def __init__(self, depth, pretrained=True, cut_at_pooling=False, train_layers="conv5", matconvnet=None):
        super().__init__()
        if depth != 16:
            raise KeyError("Unsupported depth:", depth)
        self.pretrained = pretrained
        self.depth = depth
        self.cut_at_pooling = cut_at_pooling
        self.train_layers = train_layers
        self.feature_dim = 512
        self.matconvnet = matconvnet
        layers = []
        for item in VGG16_PLAN:
            if item == "P":
                layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
            else:
                _, cin, cout = item
                layers.append(nn.Conv2d(cin, cout, kernel_size=3, padding=1))
                layers.append(nn.ReLU(inplace=True))
        self.base = nn.Sequential(*layers[:-1])  # no ReLU after conv5_3 (vgg.py:41-42)
        self.gap = nn.AdaptiveMaxPool2d(1)
        self.register_load_state_dict_post_hook(lambda module, incompatible: invalidate_caches())
        if pretrained:
            self._load_imagenet()
        self._init_params()
        if not pretrained:
            self.reset_params()
        else:
            for layer in list(self.base.children())[: self._fix_layers[train_layers]]:
                for p in layer.parameters():
                    p.requires_grad = False

    def _load_imagenet(self):
        # The reference calls torchvision.models.vgg16(pretrained=True) (vgg.py:40), a download.
        import os
        try:
            import torchvision
            tv = torchvision.models.vgg16(weights="IMAGENET1K_V1")
        except Exception as exc:  # no network on the build / GPU boxes
            if os.environ.get("IBL_VGG16_RANDOM_INIT_OK") == "1":
                # explicit opt-in for callers that load a checkpoint right after construction
                # (examples/test.py:59,97-99 builds models.create('vgg16') and then copies the checkpoint in)
                import warnings
                warnings.warn("vgg16(pretrained=True): ImageNet weights unavailable, continuing with random "
                              "init because IBL_VGG16_RANDOM_INIT_OK=1 -- load a checkpoint before use")
                self.reset_params()
                return
            raise RuntimeError(
                "vgg16(pretrained=True) needs the torchvision ImageNet weights (a download); "
                "pass pretrained=False and load a checkpoint instead, or set IBL_VGG16_RANDOM_INIT_OK=1 if a "
                "checkpoint is loaded right after construction") from exc
        sd = {k: v for k, v in tv.features.state_dict().items() if int(k.split(".")[0]) <= 28}
        self.base.load_state_dict(sd)

    def _init_params(self):
        if self.matconvnet is not None:
            self.base.load_state_dict(torch.load(self.matconvnet))
            self.pretrained = True
        invalidate_caches()

    def reset_params(self):
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out")
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
        invalidate_caches()

    def conv_params(self):
        convs = [m for m in self.base if isinstance(m, nn.Conv2d)]
        return [c.weight for c in convs], [c.bias for c in convs]

    def _bind(self, x: torch.Tensor) -> Engine:
        eng = Engine.get(x.device)
        ws, bs = self.conv_params()
        # training mode: parameters change every step, possibly through `.data` (no version bump) -> always
        # re-lay them out (25 us of device time); eval mode trusts the (address, version) key
        eng.set_vgg16(ws, bs, force=self.training and any(w.requires_grad for w in ws))
        return eng

    def first_trainable_layer(self):
        """Index (0..12) of the first conv layer with a trainable parameter, or 13 if the trunk is frozen."""
        ws, bs = self.conv_params()
        for i, (w, b) in enumerate(zip(ws, bs)):
            if w.requires_grad or b.requires_grad:
                return i
        return 13

    def forward(self, x):
        eng = self._bind(x)
        first = self.first_trainable_layer() if (self.training and torch.is_grad_enabled()) else 13
        if first < 13:
            # training: the suffix [first, 12] is differentiated (vgg.py:50-53 freezes the prefix for 'conv5' etc.)
            ws, bs = self.conv_params()
            flat = [t for l in range(first, 13) for t in (ws[l], bs[l])]
            feat = _VGGTrunkFunction.apply(x, first, *flat)
            if self.cut_at_pooling:
                return feat
            return torch.nn.functional.adaptive_max_pool2d(feat, 1).view(feat.size(0), -1), feat
        _, feat, pool = eng.vgg16_forward(x, want_nchw=True, want_pool=not self.cut_at_pooling)
        if self.cut_at_pooling:
            return feat
        return pool, feat


def vgg16(**kwargs):
    return VGG(16, **kwargs)


class NetVLAD(nn.Module):
    """Reference ibl/models/netvlad.py:8-61: forward returns the un-normalised [N,K,C] VLAD."""

    def __init__(self, num_clusters=64, dim=512, alpha=100.0, normalize_input=True):
        super().__init__()
        self.num_clusters = num_clusters
        self.dim = dim
        self.alpha = alpha
        self.normalize_input = normalize_input
        self.conv = nn.Conv2d(dim, num_clusters, kernel_size=(1, 1), bias=False)
        self.centroids = nn.Parameter(torch.rand(num_clusters, dim), requires_grad=True)
        self.clsts = None
        self.traindescs = None

    def _init_params(self):
        # netvlad.py:34-42: alpha from the mean gap between the two largest cluster responses
        import numpy as np
        assign = self.clsts / np.linalg.norm(self.clsts, axis=1, keepdims=True)
        dots = np.dot(assign, self.traindescs.T)
        dots.sort(0)
        top2 = dots[::-1, :][:2]
        self.alpha = (-np.log(0.01) / np.mean(top2[0] - top2[1])).item()
        self.centroids.data.copy_(torch.from_numpy(self.clsts))
        self.conv.weight.data.copy_(torch.from_numpy(self.alpha * assign).unsqueeze(2).unsqueeze(3))
        invalidate_caches()

    def forward(self, x):
        if torch.is_grad_enabled() and (x.requires_grad or self.conv.weight.requires_grad or self.centroids.requires_grad):
            # training (SFRS region branch, netvlad.py:139-146): forward and backward both in libiblb200
            return _NetVLADFunction.apply(x, self.conv.weight, self.centroids, self.normalize_input)
        eng = Engine.get(x.device)
        raw, _ = eng.netvlad_forward(x, self.conv.weight, self.centroids, nhwc=False,
                                     normalize_input=self.normalize_input, want_raw=True, want_norm=False)
        return raw


class _NetVLADFunction(torch.autograd.Function):
    """autograd bridge for NetVLAD: ibl_netvlad_forward / ibl_netvlad_backward (SURVEY 8 row a11)."""

    @staticmethod
    def forward(ctx, x, conv_w, centroids, normalize_input):
        eng = Engine.get(x.device)
        xc = x.contiguous()
        raw, _ = eng.netvlad_forward(xc, conv_w, centroids, nhwc=False, normalize_input=normalize_input,
                                     want_raw=True, want_norm=False)
        ctx.save_for_backward(xc, conv_w, centroids)
        ctx.normalize_input = normalize_input
        return raw

    @staticmethod
    def backward(ctx, grad_out):
        x, conv_w, centroids = ctx.saved_tensors
        eng = Engine.get(x.device)
        dx, dw, dc = eng.netvlad_backward(x, conv_w, centroids, grad_out.contiguous(), nhwc=False,
                                          normalize_input=ctx.normalize_input)
        return dx, dw.view_as(conv_w), dc, None


class _PCALayerFunction(torch.autograd.Function):
    """autograd bridge for EmbedNetPCA.pca_layer without its L2 (netvlad.py:105-107): y = v W^T + b forward
    (ibl_pca_forward_train), dgrad / wgrad / bias gradient backward (ibl_pca_backward, tensor-core wgmma kernels).  The
    gradient of the weight comes back as [P, D, 1, 1], the conv's own layout."""

    @staticmethod
    def forward(ctx, v, weight, bias):
        eng = Engine.get(v.device)
        vc = v.contiguous()
        y = eng.pca_forward_train(vc, weight, bias)
        ctx.save_for_backward(vc, weight, bias)
        return y

    @staticmethod
    def backward(ctx, gy):
        v, weight, bias = ctx.saved_tensors
        eng = Engine.get(gy.device)
        need_gv, need_gw, need_gb = ctx.needs_input_grad
        if need_gv:
            eng.set_pca(weight, bias)     # a no-op unless another PCA layer was bound since the forward
        gv, gw, gb = eng.pca_backward(v, weight, gy.contiguous(), need_gv=need_gv, need_gw=need_gw, need_gb=need_gb)
        return gv, (gw.view_as(weight) if need_gw else None), gb


class _EmbedBase(nn.Module):
    def __init__(self, base_model, net_vlad):
        super().__init__()
        self.base_model = base_model
        self.net_vlad = net_vlad
        # load_state_dict copies with Tensor.copy_ (bumps the version) but be explicit: a freshly loaded
        # checkpoint must never be served from stale re-laid-out weights
        self.register_load_state_dict_post_hook(lambda module, incompatible: invalidate_caches())

    def _init_params(self):
        self.base_model._init_params()
        self.net_vlad._init_params()

    def _bind(self, x: torch.Tensor) -> Engine:
        eng = self.base_model._bind(x)
        eng.set_netvlad(self.net_vlad.conv.weight, self.net_vlad.centroids)
        return eng

    def _train_forward(self, x):
        # differentiable path (netvlad_img.py training): trunk suffix + NetVLAD in libiblb200 through their
        # autograd Functions, the two normalisations (netvlad.py:78-80) as torch ops on [B,64,512]
        pool_x, feat = self.base_model(x)
        v = torch.nn.functional.normalize(self.net_vlad(feat), p=2, dim=2)
        return pool_x, torch.nn.functional.normalize(v.view(x.size(0), -1), p=2, dim=1)


class EmbedNet(_EmbedBase):
    """netvlad.py:63-82: forward -> (pool_x [B,512], vlad_x [B,K*C]) with intra-norm + L2."""

    def forward(self, x):
        if self.training and torch.is_grad_enabled():
            return self._train_forward(x)
        eng = self._bind(x)
        vlad, pool = eng.extract(x, pca=False, want_pool=True)
        return pool, vlad


class EmbedNetPCA(_EmbedBase):
    """netvlad.py:84-110: + 1x1 conv PCA-whitening layer and L2 -> [B,dim]."""

    def __init__(self, base_model, net_vlad, dim=4096):
        super().__init__(base_model, net_vlad)
        self.pca_layer = nn.Conv2d(net_vlad.num_clusters * net_vlad.dim, dim, 1, stride=1, padding=0)

    def _train_forward(self, x):
        # differentiable path: trunk suffix + NetVLAD + the two normalisations as EmbedNet._train_forward, then the PCA
        # layer through its autograd Function and the final L2 (netvlad.py:95-110).  Parameters change every step,
        # possibly through `.data`, so the weight planes are re-laid out every time (as VGG._bind does for the trunk).
        _, v = super()._train_forward(x)
        Engine.get(x.device).set_pca(self.pca_layer.weight, self.pca_layer.bias, force=True)
        y = _PCALayerFunction.apply(v, self.pca_layer.weight, self.pca_layer.bias)
        return torch.nn.functional.normalize(y, p=2, dim=-1)

    def forward(self, x):
        if self.training and torch.is_grad_enabled():
            return self._train_forward(x)
        eng = self._bind(x)
        eng.set_pca(self.pca_layer.weight, self.pca_layer.bias)
        out, _ = eng.extract(x, pca=True, want_pool=False)
        return out


class EmbedRegionNet(_EmbedBase):
    """netvlad.py:112-207.  Eval: (pool, vlad) like EmbedNet (:199-205).  Train: the SFRS region branch
    (:123-194) -- quarter / half / global region VLADs of the anchor and of every pair image and their 9x9
    similarity matrix.  NetVLAD and the trainable part of the VGG trunk run forward and backward in libiblb200."""

    def __init__(self, base_model, net_vlad, tuple_size=1):
        super().__init__(base_model, net_vlad)
        self.tuple_size = tuple_size

    @staticmethod
    def _quarters(feat):
        # [N,C,H,W] -> [N*4,C,H/2,W/2], region order (top-left, top-right, bottom-left, bottom-right)
        N, C, H, W = feat.shape
        h2, w2 = H // 2, W // 2
        q = feat[:, :, : 2 * h2, : 2 * w2].reshape(N, C, 2, h2, 2, w2).permute(0, 2, 4, 1, 3, 5)
        return q.reshape(N * 4, C, h2, w2).contiguous()

    def _region_descriptors(self, feat):
        # -> [N, 9, K*C]: global, 4 halves (top, bottom, left, right), 4 quarters; intra-norm + L2 each
        N = feat.shape[0]
        quarter = self.net_vlad(self._quarters(feat))                       # [(N*4), K, C]
        K, C = quarter.shape[1:]
        quarter = quarter.view(N, 4, K, C)
        half = torch.stack((quarter[:, 0] + quarter[:, 1], quarter[:, 2] + quarter[:, 3],
                            quarter[:, 0] + quarter[:, 2], quarter[:, 1] + quarter[:, 3]), dim=1)
        whole = quarter.sum(dim=1, keepdim=True)
        v = torch.cat((whole, half, quarter), dim=1)                        # [N, 9, K, C]
        v = torch.nn.functional.normalize(v, p=2, dim=3).reshape(N, 9, K * C)
        return torch.nn.functional.normalize(v, p=2, dim=2)

    def _forward_train(self, feat):
        B, C, H, W = feat.shape
        t = feat.view(self.tuple_size, -1, C, H, W)
        anchors = t[:, 0].contiguous()                                      # [T,C,H,W]
        pairs = t[:, 1:].reshape(-1, C, H, W)                               # [T*(n-1),C,H,W]
        va = self._region_descriptors(anchors).view(self.tuple_size, 1, 9, -1)
        vb = self._region_descriptors(pairs).view(self.tuple_size, -1, 9, va.shape[-1])
        score = torch.matmul(va, vb.transpose(2, 3))                        # [T, n-1, 9, 9] (anchor broadcast)
        return score, va, vb

    def forward(self, x):
        if not self.training:
            eng = self._bind(x)
            vlad, pool = eng.extract(x, pca=False, want_pool=True)
            return pool, vlad
        _, feat = self.base_model(x)          # differentiable through the trainable suffix of the trunk
        return self._forward_train(feat)


_factory = {
    "vgg16": vgg16,
    "netvlad": NetVLAD,
    "embednet": EmbedNet,
    "embednetpca": EmbedNetPCA,
    "embedregionnet": EmbedRegionNet,
}


def names():
    return sorted(_factory.keys())


def create(name, *args, **kwargs):
    """Same contract as ibl/models/__init__.py:20-53."""
    if name not in _factory:
        raise KeyError("Unknown model:", name)
    return _factory[name](*args, **kwargs)
