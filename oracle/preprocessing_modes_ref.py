"""TEST INFRASTRUCTURE ONLY (never imported by pytracking_b200/): the border modes 'inside' and 'inside_major' of the reference's crop
sampling (pytracking/features/preprocessing.py:76-124), restated on top of oracle/preprocessing_ref.py with the same split into a
float32 *geometry* step (what csrc/dimp_tracker.cu `plan_patch` computes on the host) and a *resampling* step (what
`sample_patch_kernel` computes on the device).  Padding stays 'replicate' in every mode.
Pinned: oracle/gen_prdimp_golden.py asserts bit-equality with the reference's `sample_patch` on every recorded PrDiMP frame.
"""
import torch
import torch.nn.functional as F

from oracle import preprocessing_ref as R

MODES = ("replicate", "inside", "inside_major")


def sample_patch_geometry(im, pos, sample_sz, output_sz, mode="replicate", max_scale_change=None):
    """-> (df, os_r, os_c, tl_r, tl_c, in_h, in_w, patch_coord[1,4] float32), torch's types as preprocessing.py:72-137 has them:
    im_sz float32, the shrink clamp, `.long()` truncation of the shrunk size before the decimation factor, float32 tl / br, the two
    shift steps with clamp(0), float floor division and (outside > 0).long()."""
    if mode not in MODES:
        raise NotImplementedError(mode)
    if mode == "replicate":
        return R.sample_patch_geometry(im, pos, sample_sz, output_sz)
    posl = pos.long().clone()
    im_sz = torch.Tensor([im.shape[2], im.shape[3]])
    shrink = sample_sz.float() / im_sz
    shrink = shrink.max() if mode == "inside" else shrink.min()
    shrink.clamp_(min=1, max=max_scale_change)
    sample_sz = (sample_sz.float() / shrink).long()
    df = max(int(torch.min(sample_sz.float() / output_sz.float()).item() - 0.1), 1)
    sz = sample_sz.float() / df
    offs = torch.zeros(2, dtype=torch.long)
    if df > 1:
        offs = posl % df
        posl = (posl - offs) / df
    im2_sz = torch.LongTensor([len(range(int(offs[0]), im.shape[2], df)), len(range(int(offs[1]), im.shape[3], df))])
    szl = torch.max(sz.round(), torch.Tensor([2])).long()
    tl = posl - (szl - 1) / 2
    br = posl + szl / 2 + 1
    shift = (-tl).clamp(0) - (br - im2_sz).clamp(0)
    tl += shift
    br += shift
    outside = ((-tl).clamp(0) + (br - im2_sz).clamp(0)) // 2
    shift = (-tl - outside) * (outside > 0).long()
    tl += shift
    br += shift
    lo_i, hi_i = tl.int(), br.int()
    coord = df * torch.cat((tl, br)).view(1, 4)
    return (df, int(offs[0]), int(offs[1]), int(lo_i[0]), int(lo_i[1]), int(hi_i[0] - lo_i[0]), int(hi_i[1] - lo_i[1]), coord)


def sample_patch(im, pos, sample_sz, output_sz=None, mode="replicate", max_scale_change=None):
    """-> (patch [1,C,h,w], patch_coord [1,4]); replicate padding is a clamped gather of the decimated image."""
    df, os_r, os_c, tl_r, tl_c, in_h, in_w, coord = sample_patch_geometry(im, pos, sample_sz, output_sz, mode, max_scale_change)
    dec = im[..., os_r::df, os_c::df]
    rows = (torch.arange(in_h) + tl_r).clamp(0, dec.shape[-2] - 1)
    cols = (torch.arange(in_w) + tl_c).clamp(0, dec.shape[-1] - 1)
    patch = dec[..., rows, :][..., cols]
    if output_sz is None or (patch.shape[-2] == output_sz[0] and patch.shape[-1] == output_sz[1]):
        return patch.clone(), coord
    return F.interpolate(patch, output_sz.long().tolist(), mode="bilinear"), coord
