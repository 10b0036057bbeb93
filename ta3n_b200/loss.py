"""Loss heads that follow the path in the reference's training step (SURVEY §8f, row n1).

torch-op versions with the reference's semantics; they consume the outputs of VideoModel.forward
and stay differentiable through the fused operator.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def cross_entropy_soft(pred):
    """loss.py:8-12 -- mean entropy of softmax(pred)."""
    return torch.mean(torch.sum(-F.softmax(pred, dim=1) * F.log_softmax(pred, dim=1), 1))


def attentive_entropy(pred, pred_domain):
    """loss.py:15-25 -- entropy of the class prediction weighted by (1 + domain entropy)."""
    dom_ent = torch.sum(-F.softmax(pred_domain, dim=1) * F.log_softmax(pred_domain, dim=1), 1)
    cls_ent = torch.sum(-F.softmax(pred, dim=1) * F.log_softmax(pred, dim=1), 1)
    return torch.mean((1 + dom_ent) * cls_ent)


def dis_MCD(out1, out2):
    """loss.py:29-30 -- classifier discrepancy of the MCD variant (main.py:548-556): mean |softmax(out1) - softmax(out2)|."""
    return torch.mean(torch.abs(F.softmax(out1, dim=1) - F.softmax(out2, dim=1)))


def ta3n_loss(outputs, label_source, gamma=0.003, place_adv=('Y', 'Y', 'Y'), use_attn='TransAttn',
              add_loss_DA='attentive_entropy', use_target='uSv', label_target=None):
    """Loss of the shipped configuration (adv_DA='RevGrad'):
    main.py:446 (source CE) + main.py:508-538 (domain CE per level) + main.py:541-545 (target entropy; 0 without a
    target row) or main.py:559-562 (attentive entropy).
    use_target: 'uSv' (default) as above; 'Sv' takes the class CE over cat(out_source, out_target) against
    cat(label_source, label_target) (main.py:442-446), every other term unchanged; 'none' is the CE of the source rows
    alone (main.py guards every DA term with use_target != 'none')."""
    (_, out_s, _, pd_s, _, _, out_t, _, pd_t, _) = outputs
    if use_target not in ('uSv', 'Sv', 'none'):
        raise ValueError(f"use_target must be 'uSv', 'Sv' or 'none', got {use_target!r}")
    if use_target == 'none':
        return F.cross_entropy(out_s, label_source)
    if use_target == 'Sv':
        if label_target is None or tuple(label_target.shape) != (out_t.size(0),):
            raise ValueError(f"use_target='Sv' needs label_target with one label per target row ({out_t.size(0)})")
        loss = F.cross_entropy(torch.cat([out_s, out_t], 0), torch.cat([label_source, label_target], 0))
    else:
        loss = F.cross_entropy(out_s, label_source)
    per_level = []
    for lvl, flag in enumerate(place_adv):
        if flag != 'Y':
            continue
        ps, pt = pd_s[lvl].reshape(-1, 2), pd_t[lvl].reshape(-1, 2)
        dom = torch.cat([torch.zeros(ps.size(0), dtype=torch.long, device=ps.device),
                         torch.ones(pt.size(0), dtype=torch.long, device=pt.device)])
        both = torch.cat([ps, pt], 0)
        per_level.append(both)
        loss = loss + F.cross_entropy(both, dom)
    if add_loss_DA == 'target_entropy' and out_t.size(0) > 0:
        loss = loss + gamma * cross_entropy_soft(out_t)
    if add_loss_DA == 'attentive_entropy' and use_attn != 'none' and len(per_level) > 1:
        loss = loss + gamma * attentive_entropy(torch.cat([out_s, out_t], 0), per_level[1])
    return loss


# ---- discrepancy-based alignment, --dis_DA DAN / JAN (main.py:455-505, loss.py:46-120) ------------------------------
_DIS_CHUNK = 256        # main.py:487: DAN computes each level over chunks of at most this many rows per domain


def guassian_kernel(source, target, kernel_mul=2.0, kernel_num=5, fix_sigma=None):
    """loss.py:46-58 (the reference's spelling) -- the sum of ``kernel_num`` Gaussian kernels over the rows of
    cat(source, target): exp(-||x_i - x_j||^2 / (bw * kernel_mul^k)), k < kernel_num.  bw = fix_sigma, or the mean
    off-diagonal squared distance, taken detached, divided by kernel_mul^(kernel_num // 2)."""
    rows = torch.cat([source, target], 0)
    n = rows.size(0)
    l2 = ((rows.unsqueeze(0) - rows.unsqueeze(1)) ** 2).sum(2)
    bw = fix_sigma if fix_sigma else torch.sum(l2.detach()) / (n * n - n)
    bw = bw / kernel_mul ** (kernel_num // 2)
    return sum(torch.exp(-l2 / (bw * kernel_mul ** k)) for k in range(kernel_num))


def _mmd_from_kernels(k, n, ver):
    """The MMD estimate of loss.py:60-80 / 99-118 from the (2n, 2n) kernel matrix of cat(source, target)."""
    if ver == 2:
        return torch.mean(k[:n, :n] + k[n:, n:] - k[:n, n:] - k[n:, :n])
    if ver == 1:
        i = torch.arange(n, device=k.device)
        j = (i + 1) % n
        terms = k[i, j] + k[i + n, j + n] - k[i, j + n] - k[j, i + n]
        return terms.sum().abs() / float(n)
    raise ValueError('ver == 1 or 2')


def mmd_rbf(source, target, kernel_mul=2.0, kernel_num=5, fix_sigma=None, ver=2):
    """loss.py:60-80 -- multi-kernel MMD between equal-sized source and target batches (DAN)."""
    k = guassian_kernel(source, target, kernel_mul=kernel_mul, kernel_num=kernel_num, fix_sigma=fix_sigma)
    return _mmd_from_kernels(k, int(source.size(0)), ver)


def JAN(source_list, target_list, kernel_muls=[2.0, 2.0], kernel_nums=[2, 5], fix_sigma_list=[None, None], ver=2):  # noqa: B006,N802
    """loss.py:82-120 -- joint MMD: the product of the layers' kernel matrices, then the MMD estimate."""
    joint = None
    for i, (s, t) in enumerate(zip(source_list, target_list)):
        k = guassian_kernel(s, t, kernel_mul=kernel_muls[i], kernel_num=kernel_nums[i], fix_sigma=fix_sigma_list[i])
        joint = k if joint is None else joint * k
    return _mmd_from_kernels(joint, int(source_list[0].size(0)), ver)


def discrepancy_loss(feat_source, feat_target, dis_DA, add_fc=1, place_dis=('Y', 'Y', 'N')):  # noqa: N803
    """``loss_discrepancy`` of main.py:455-504 (without alpha: main.py:505 adds alpha times it to the loss).
    ``feat_source`` / ``feat_target``: the reversed feature lists of VideoModel's output with the padded rows removed,
    [pred_video, feat_video, feat_fc_L, ..., feat_fc_1].  Both sides use their first min(source rows, target rows) rows.

    DAN: the sum over the levels l < add_fc + 2 with place_dis[l] == 'Y' of the mean of mmd_rbf (kernel_mul 2,
    kernel_num 2 for the logits, 5 after) over chunks of min(256, rows) rows.  JAN: JAN over [pred_video, feat_video].

    Where the reference fails, this returns 0: no target row, or (DAN) more than 256 rows that 256 does not divide.
    A level on a 3-D shared-layer feature (l >= 2), a place_dis shorter than add_fc + 2 and an unknown dis_DA raise
    ValueError; 'CORAL' raises NotImplementedError (main.py:493 calls a CORAL the reference never defines)."""
    if dis_DA == 'CORAL':
        raise NotImplementedError("dis_DA='CORAL': the reference calls a CORAL loss it does not define")
    if dis_DA not in ('DAN', 'JAN'):
        raise ValueError(f"dis_DA must be 'DAN' or 'JAN', got {dis_DA!r}")
    n = min(feat_source[0].size(0), feat_target[0].size(0))
    zero = feat_source[0].new_zeros(())
    if dis_DA == 'JAN':
        if n == 0:
            return zero
        return JAN([f[:n] for f in feat_source[:2]], [f[:n] for f in feat_target[:2]], kernel_muls=[2.0, 2.0],
                   kernel_nums=[2, 5], fix_sigma_list=[None, None], ver=2)
    levels = dis_levels(place_dis, add_fc)
    if n == 0 or (n > _DIS_CHUNK and n % _DIS_CHUNK):
        return zero
    size = min(_DIS_CHUNK, n)
    loss = zero
    for lvl in levels:
        xs, xt = feat_source[lvl][:n], feat_target[lvl][:n]
        chunks = [mmd_rbf(xs[c:c + size], xt[c:c + size], kernel_mul=2.0, kernel_num=2 if lvl == 0 else 5, ver=2)
                  for c in range(0, n, size)]
        loss = loss + sum(chunks) / len(chunks)
    return loss


def dis_levels(place_dis, add_fc=1):
    """The DAN levels of main.py:478-479: l < add_fc + 2 with place_dis[l] == 'Y'.  Only the logits (0) and the video
    feature (1) are 2-D; the reference fails on the 3-D shared-layer levels, so they, a place_dis shorter than
    add_fc + 2 and a place_dis with no level (the reference then calls .item() on the integer 0) raise ValueError."""
    if len(place_dis) < add_fc + 2:
        raise ValueError(f"place_dis needs add_fc + 2 = {add_fc + 2} entries, got {len(place_dis)}")
    levels = [lvl for lvl in range(add_fc + 2) if place_dis[lvl] == 'Y']
    if any(lvl >= 2 for lvl in levels):
        raise ValueError("place_dis[l] == 'Y' for l >= 2: the shared-layer features are 3-D, which the reference's "
                         "gaussian kernel does not take")
    if not levels:
        raise ValueError(f"place_dis {tuple(place_dis)} selects no level: DAN needs 'Y' at level 0 (logits) or 1 "
                         "(video feature)")
    return levels
