"""Seeded inputs and the two references shared by the mask-loss tests (tests/test_gpu_mask_loss.py,
tests/test_mask_loss_host.py) and tools/time_mask_loss.py.

  * `clustered_inputs`: FCOS-like positives, several jittered boxes per object, COCO-like object sizes, on one batch;
  * `composition`: SipMaskHead.loss's block (sipmask_head.py:446-463) as the reference runs it on the device: fp32
    matmuls, sigmoid, CropSplit / CropSplitGt (ops.crop_split / crop_split_gt, bit for bit the reference kernels),
    F.binary_cross_entropy, the per-instance normalisation and weighting;
  * `reference64`: the same loss and its gradients in float64, dz written out (no saturation for |z| < 15).
"""
import numpy as np
import torch
import torch.nn.functional as F


def pack_bits(planes):
    """{0, 1} planes [G, H, W] -> [G, H, ceil(W / 32)] int32 words, bit x % 32 of word x / 32 is pixel x"""
    p = np.asarray(planes, dtype=bool)
    G, H, W = p.shape
    words = (W + 31) // 32
    pad = np.zeros((G, H, words * 32), dtype=bool)
    pad[:, :, :W] = p
    w = np.packbits(pad, axis=-1, bitorder='little').view('<u4')
    return torch.from_numpy(np.ascontiguousarray(w).view(np.int32))


def clustered_inputs(B, H, W, per_img, seed, grid=True, zmax=14.0, objs_per_img=None):
    """One batch: feat [B, 32, H, W], cofs [M, 128], boxes [M, 4] (mask coordinates), img_offsets [B + 1] int32, gt
    planes [G, H, W] float {0, 1} at the mask resolution, gt_rows [M] int64, weights [M].  Positives come in clusters:
    each object (COCO-like size, log-uniform 8 .. H / 2 mask pixels) gets several boxes jittered by up to 15 %.
    grid=True: feat and cofs on a 2^-8 grid with |feat| <= 1 and |cof| <= zmax / 32, so every 32-term dot product is
    exact in fp32 in any order and |z| <= zmax.  grid=False: the same bound, unrounded fp32 values."""
    rs = np.random.RandomState(seed)
    n_objs = objs_per_img or max(1, per_img // 6)
    cmax = zmax / 32.0
    feat = rs.uniform(-1, 1, (B, 32, H, W))
    cofs, boxes, rows, weights, planes, offs = [], [], [], [], [], [0]
    for b in range(B):
        objs = []
        for _ in range(n_objs):
            s = np.exp(rs.uniform(np.log(8), np.log(max(9, min(H, W) / 2))))
            ar = np.exp(rs.uniform(-0.7, 0.7))
            w_, h_ = s * ar, s / ar
            cx, cy = rs.uniform(0, W), rs.uniform(0, H)
            objs.append((cx - w_ / 2, cy - h_ / 2, cx + w_ / 2, cy + h_ / 2))
            yy, xx = np.mgrid[0:H, 0:W]
            ell = ((xx - cx) / (w_ / 2)) ** 2 + ((yy - cy) / (h_ / 2)) ** 2 <= 1.0
            planes.append(ell.astype(np.float32))
        g0 = len(planes) - n_objs
        for _ in range(per_img):
            o = rs.randint(n_objs)
            x1, y1, x2, y2 = objs[o]
            bw, bh = x2 - x1, y2 - y1
            j = rs.uniform(-0.15, 0.15, 4) * np.array([bw, bh, bw, bh])
            bx = np.array([x1, y1, x2, y2]) + j
            bx[2] = max(bx[2], bx[0] + 1.5)
            bx[3] = max(bx[3], bx[1] + 1.5)
            boxes.append(bx)
            rows.append(g0 + o)
            cofs.append(rs.uniform(-cmax, cmax, 128))
            weights.append(rs.uniform(0.2, 1.8))
        offs.append(offs[-1] + per_img)
    feat = torch.tensor(feat, dtype=torch.float32)
    cofs = torch.tensor(np.array(cofs).reshape(-1, 128), dtype=torch.float32)
    if grid:
        feat = torch.round(feat * 256) / 256
        cofs = torch.clamp(torch.round(cofs * 256) / 256, -cmax, cmax)
    return dict(feat=feat, cofs=cofs, boxes=torch.tensor(np.array(boxes).reshape(-1, 4), dtype=torch.float32),
                offsets=torch.tensor(offs, dtype=torch.int32),
                planes=torch.tensor(np.array(planes).reshape(-1, H, W), dtype=torch.float32),
                rows=torch.tensor(rows, dtype=torch.int64), weights=torch.tensor(weights, dtype=torch.float32))


def to_device(inp, device='cuda'):
    out = {k: v.to(device) for k, v in inp.items()}
    out['bits'] = pack_bits(inp['planes'].numpy()).to(device)
    return out


def composition(inp, feat, cofs, crop_split_fn, crop_split_gt_fn, keep_dz=None):
    """loss [B] of the reference's per-image block on the device, differentiable w.r.t. `feat` and `cofs` (used in place of
    inp['feat'] / inp['cofs']).  keep_dz: a list that receives each image's stacked logits Z [4, H, W, M_b] with
    retain_grad(), so that dZ can be read after backward."""
    offs = inp['offsets'].tolist()
    planes, rows, boxes, weights = inp['planes'], inp['rows'], inp['boxes'], inp['weights']
    losses = []
    for b in range(feat.shape[0]):
        n0, n1 = offs[b], offs[b + 1]
        if n1 == n0:
            losses.append(feat[b].sum() * 0)
            continue
        img_mask1 = feat[b].permute(1, 2, 0)
        cof = cofs[n0:n1]
        z = torch.stack([img_mask1 @ cof[:, 32 * q:32 * q + 32].t() for q in range(4)], dim=0)
        if keep_dz is not None:
            z.retain_grad()
            keep_dz.append(z)
        pred = crop_split_fn(torch.sigmoid(z).contiguous(), boxes[n0:n1])
        gt = planes.index_select(0, rows[n0:n1]).permute(1, 2, 0).contiguous()
        gt_crop = crop_split_gt_fn(gt, boxes[n0:n1])
        pre = F.binary_cross_entropy(pred, gt_crop, reduction='none')
        bx = boxes[n0:n1]
        bw, bh = bx[:, 2] - bx[:, 0], bx[:, 3] - bx[:, 1]
        pre = pre.sum(dim=(0, 1)) / bw / bh / (n1 - n0)
        losses.append(torch.sum(pre * weights[n0:n1]))
    return torch.stack(losses)


def cells(boxes, H, W):
    """[M, H, W] int64: the CropSplit cell of each pixel (crop_split_cuda_kernel.cu:44-53, fp32 geometry), -1 outside"""
    b = boxes.float()
    x1, y1, x2, y2 = [b[:, i].view(-1, 1, 1) for i in range(4)]
    roi_w = (((x2 - x1).double() + 0.1) / 2).float()
    roi_h = (((y2 - y1).double() + 0.1) / 2).float()
    hh = torch.arange(H, dtype=torch.float32, device=b.device).view(1, -1, 1)
    ww = torch.arange(W, dtype=torch.float32, device=b.device).view(1, 1, -1)
    inside = (ww >= x1) & (hh >= y1) & (ww < x2) & (hh < y2)
    cell = (torch.trunc((hh - y1) / roi_h) * 2 + torch.trunc((ww - x1) / roi_w)).clamp(0, 3).long()
    return torch.where(inside, cell, torch.full_like(cell, -1))


def reference64(inp, g=None):
    """float64 loss [B], d feat [B, 32, H, W] and d cofs [M, 128] for upstream gradient g [B] (ones by default), with
    the fp32 cell geometry; dz = c (p - t) (the BCE backward through the sigmoid without the clamp, exact for |z| < 15)."""
    feat, cofs, boxes = inp['feat'].double(), inp['cofs'].double(), inp['boxes']
    B, _, H, W = feat.shape
    offs = inp['offsets'].tolist()
    g = torch.ones(B, dtype=torch.float64) if g is None else g.double().cpu()
    loss = torch.zeros(B, dtype=torch.float64)
    dfeat = torch.zeros_like(feat)
    dcofs = torch.zeros_like(cofs)
    for b in range(B):
        n0, n1 = offs[b], offs[b + 1]
        if n1 == n0:
            continue
        Mb = n1 - n0
        X = feat[b].reshape(32, -1).t()                                            # [HW, 32]
        cl = cells(boxes[n0:n1], H, W).reshape(Mb, -1).t().to(feat.device)         # [HW, Mb]
        C = cofs[n0:n1].view(Mb, 4, 32)
        zq = torch.einsum('pk,nqk->pnq', X, C)                                     # [HW, Mb, 4]
        z = torch.gather(zq, 2, cl.clamp(min=0).unsqueeze(-1)).squeeze(-1)
        t = inp['planes'].double().to(feat.device).index_select(0, inp['rows'][n0:n1].to(feat.device))
        t = t.reshape(Mb, -1).t()
        p = torch.sigmoid(z)
        term = -(t * torch.log(p).clamp(min=-100) + (1 - t) * torch.log1p(-p).clamp(min=-100))
        inside = (cl >= 0).double()
        bx = boxes[n0:n1].double().to(feat.device)
        area = (bx[:, 2] - bx[:, 0]) * (bx[:, 3] - bx[:, 1])
        coef = inp['weights'][n0:n1].double().to(feat.device) / area / Mb
        loss[b] = (term * inside * coef).sum()
        dz = g[b] * coef * (p - t) * inside                                        # [HW, Mb]
        onehot = F.one_hot(cl.clamp(min=0), 4).double() * inside.unsqueeze(-1)     # [HW, Mb, 4]
        dzq = dz.unsqueeze(-1) * onehot
        dfeat[b] = torch.einsum('pnq,nqk->pk', dzq, C).t().reshape(32, H, W)
        dcofs[n0:n1] = torch.einsum('pnq,pk->nqk', dzq, X).reshape(Mb, 128)
    return loss, dfeat, dcofs
