"""Host-side mirror of the reference's training steps (ibl/trainers.py):

* `Trainer` (trainers.py:11-162): NetVLAD (triplet loss) and SARE (`sare_ind` / `sare_joint`) training of `EmbedNet`
  (or of the bare `VGG` with max pooling, `vlad=False`), as examples/netvlad_img.py drives it;
* `SFRSTrainer` (trainers.py:165-320): the SFRS step, with the same constructor, `train`, `_parse_data`, `_forward`,
  `_get_hard_loss` and `_get_loss`.

What runs where: the model forward/backward (VGG trunk suffix, NetVLAD) is libiblb200 through the autograd Functions of
openibl_b200.models; the loss algebra below works on a handful of [B, n, 32768] descriptors (and, for SFRS,
[B, n, 9, 9] similarity matrices) per step and is plain torch, as in the reference.  BASELINE configs[4] drives the
SFRS step with tuple_size = 4 under DistributedDataParallel (examples/sfrs_step_synthetic.py); tools/bench_train.py
times the `Trainer` step."""
from __future__ import annotations

import time

import torch
import torch.nn.functional as F

from .utils.meters import AverageMeter


def _rank():
    try:
        return torch.distributed.get_rank()
    except Exception:
        return 0


class Trainer(object):
    """NetVLAD (CVPR'16, loss_type='triplet') and SARE (ICCV'19, 'sare_ind' / 'sare_joint') training.

    The losses are the reference's Euclidean versions (trainers.py:90-140): the triplet margin loss on L2 distances,
    and SARE's log-softmax over negated squared distances -- not the dot-product versions `SFRSTrainer` uses.
    `_get_loss` raises ValueError for an unknown loss type (the reference's `assert ("...")` always passes and then
    fails on the unbound `loss`)."""

    def __init__(self, model, margin=0.3, gpu=None, temp=0.07):
        self.model, self.gpu, self.margin, self.temp = model, gpu, margin, temp

    # ---- one epoch (trainers.py:24-61) ------------------------------------------------------------------------
    def train(self, epoch, sub_id, data_loader, optimizer, train_iters, print_freq=1, vlad=True, loss_type="triplet"):
        self.model.train()
        batch_time, data_time, losses = AverageMeter(), AverageMeter(), AverageMeter()
        end = time.time()
        data_loader.new_epoch()
        for i in range(train_iters):
            inputs = self._parse_data(data_loader.next())
            data_time.update(time.time() - end)
            loss = self._forward(inputs, vlad, loss_type)
            losses.update(loss.item())
            optimizer.zero_grad()
            loss.backward()
            optimizer.step()
            batch_time.update(time.time() - end)
            end = time.time()
            if (i + 1) % print_freq == 0 and _rank() == 0:
                print("Epoch: [{}-{}][{}/{}]\tTime {:.3f} ({:.3f})\tData {:.3f} ({:.3f})\tLoss {:.3f} ({:.3f})".format(
                    epoch, sub_id, i + 1, train_iters, batch_time.val, batch_time.avg, data_time.val, data_time.avg,
                    losses.val, losses.avg))

    def _parse_data(self, inputs):
        """trainers.py:64-68: the collated tuple positions -> [B, N, C, H, W] on the device."""
        imgs = torch.stack([item[0] for item in inputs]).permute(1, 0, 2, 3, 4)
        return imgs.cuda(self.gpu)

    def _forward(self, inputs, vlad, loss_type):
        """trainers.py:70-80: the loss on the VLAD descriptor when `vlad`, else on the max-pooled conv5 feature."""
        B, N, C, H, W = inputs.size()
        outputs_pool, outputs_vlad = self.model(inputs.reshape(-1, C, H, W))
        return self._get_loss(outputs_vlad if vlad else outputs_pool, loss_type, B, N)

    def _get_loss(self, outputs, loss_type, B, N):
        """trainers.py:82-162.  outputs [B*N, L], tuple order (anchor, positive, N-2 negatives)."""
        outputs = outputs.reshape(B, N, -1)
        L = outputs.size(-1)
        a, p, n = outputs[:, 0], outputs[:, 1], outputs[:, 2:]
        if loss_type == "triplet":
            ae = a.unsqueeze(1).expand_as(n).reshape(-1, L)
            pe = p.unsqueeze(1).expand_as(n).reshape(-1, L)
            return F.triplet_margin_loss(ae, pe, n.reshape(-1, L), margin=self.margin, p=2, reduction="mean")
        if loss_type not in ("sare_joint", "sare_ind"):
            raise ValueError("Unknown loss function: {}".format(loss_type))
        dist_pos = ((a - p) ** 2).sum(1).view(B, 1)                                        # [B,1]
        dist_neg = ((a.unsqueeze(1).expand_as(n).reshape(-1, L) - n.reshape(-1, L)) ** 2).sum(1).view(B, -1)
        if loss_type == "sare_joint":
            logits = -torch.cat((dist_pos, dist_neg), 1)                                   # [B, 1+n]
        else:
            logits = -torch.stack((dist_pos.expand_as(dist_neg), dist_neg), 2).reshape(-1, 2)   # [B*n, 2]
        return (-F.log_softmax(logits, 1)[:, 0]).mean()


class SFRSTrainer(object):
    def __init__(self, model, model_cache, margin=0.3, neg_num=10, gpu=None, temp=[0.07, ]):
        self.model, self.model_cache = model, model_cache
        self.margin, self.gpu, self.neg_num, self.temp = margin, gpu, neg_num, temp

    # ---- one epoch (trainers.py:181-226) ----------------------------------------------------------------------
    def train(self, gen, epoch, sub_id, data_loader, optimizer, train_iters, print_freq=1, lambda_soft=0.5,
              loss_type="sare_ind"):
        self.model.train()
        self.model_cache.train()
        batch_time, data_time, losses_hard, losses_soft = AverageMeter(), AverageMeter(), AverageMeter(), AverageMeter()
        end = time.time()
        data_loader.new_epoch()
        for i in range(train_iters):
            inputs_easy, inputs_diff = self._parse_data(data_loader.next())
            data_time.update(time.time() - end)
            loss_hard, loss_soft = self._forward(inputs_easy, inputs_diff, loss_type, gen)
            loss = loss_hard + loss_soft * lambda_soft
            optimizer.zero_grad()
            loss.backward()
            optimizer.step()
            losses_hard.update(loss_hard.item())
            losses_soft.update(loss_soft.item())
            batch_time.update(time.time() - end)
            end = time.time()
            if (i + 1) % print_freq == 0 and _rank() == 0:
                print("Epoch: [{}-{}][{}/{}]\tTime {:.3f} ({:.3f})\tData {:.3f} ({:.3f})\t"
                      "Loss_hard {:.3f} ({:.3f})\tLoss_soft {:.3f} ({:.3f})".format(
                          epoch, sub_id, i + 1, train_iters, batch_time.val, batch_time.avg, data_time.val, data_time.avg,
                          losses_hard.val, losses_hard.avg, losses_soft.val, losses_soft.avg))

    def _parse_data(self, inputs):
        """trainers.py:228-233: tuple = (anchor, positive, neg_num negatives, difficult positives...)."""
        imgs = torch.stack([item[0] for item in inputs]).permute(1, 0, 2, 3, 4)
        easy = imgs[:, : self.neg_num + 2]
        diff = torch.cat((imgs[:, :1], imgs[:, self.neg_num + 2:]), dim=1)
        return easy.cuda(self.gpu), diff.cuda(self.gpu)

    # ---- losses (trainers.py:235-259) ---------------------------------------------------------------------------
    def _forward(self, inputs_easy, inputs_diff, loss_type, gen):
        B, _, C, H, W = inputs_easy.size()
        sim_easy, vlad_anchors, vlad_pairs = self.model(inputs_easy.reshape(-1, C, H, W))
        diff = inputs_diff.reshape(-1, C, H, W)
        with torch.no_grad():
            sim_diff_label, _, _ = self.model_cache(diff)      # teacher similarities, [B, diff_pos_num, 9, 9]
        sim_diff, _, _ = self.model(diff)
        if gen == 0:
            loss_hard = self._get_loss(vlad_anchors[:, 0, 0], vlad_pairs[:, 0, 0], vlad_pairs[:, 1:, 0], B, loss_type)
        else:
            per_tuple = [self._get_hard_loss(vlad_anchors[t, 0, 0], vlad_pairs[t, 0, 0], vlad_pairs[t, 1:],
                                             sim_easy[t, 1:, 0].detach(), loss_type) for t in range(B)]
            loss_hard = sum(per_tuple) / B
        # soft-label cross entropy between the teacher's and the student's image-to-region similarities (row 0)
        student = F.log_softmax(sim_diff[:, :, 0].reshape(B, -1) / self.temp[0], dim=1)
        teacher = F.softmax(sim_diff_label[:, :, 0].reshape(B, -1) / self.temp[gen], dim=1).detach()
        loss_soft = -(teacher * student).mean(0).sum()
        return loss_hard, loss_soft

    def _get_hard_loss(self, anchors, positives, negatives, score_neg, loss_type):
        """trainers.py:261-271: for every negative image keep its region most similar to the anchor image."""
        best = score_neg.reshape(self.neg_num, -1).argmax(1)                        # [neg_num]
        picked = negatives[torch.arange(negatives.size(0), device=negatives.device), best]   # [neg_num, L]
        return self._get_loss(anchors.unsqueeze(0), positives.unsqueeze(0), picked.unsqueeze(0), 1, loss_type)

    def _get_loss(self, output_anchors, output_positives, output_negatives, B, loss_type):
        """trainers.py:273-320.  anchors/positives [B,L], negatives [B,n,L]."""
        a, p, n = output_anchors, output_positives, output_negatives
        if loss_type == "triplet":
            L = a.size(-1)
            ae = a.unsqueeze(1).expand_as(n).reshape(-1, L)
            pe = p.unsqueeze(1).expand_as(n).reshape(-1, L)
            return F.triplet_margin_loss(ae, pe, n.reshape(-1, L), margin=self.margin, p=2, reduction="mean")
        sim_pos = (a * p).sum(-1, keepdim=True)                 # [B,1]   (the diagonal of anchors . positives^T)
        sim_neg = (a.unsqueeze(1) * n).sum(-1)                  # [B,n]
        if loss_type == "sare_joint":
            logits = torch.cat((sim_pos, sim_neg), 1) / self.temp[0]
            return (-F.log_softmax(logits, 1)[:, 0]).mean()
        if loss_type == "sare_ind":
            pairs = torch.stack((sim_pos.expand_as(sim_neg), sim_neg), 2).reshape(-1, 2) / self.temp[0]
            return (-F.log_softmax(pairs, 1)[:, 0]).mean()
        raise ValueError("Unknown loss function: {}".format(loss_type))
