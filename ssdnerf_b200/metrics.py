"""SSIM of rendered test views (`ssim`), and FID / KID over rendered images: the eval-side exchange of the reference (SURVEY.md §8 f3).

Surface of lib/core/evaluation/metrics.py:135-215 (`FIDKID(num_images, num_subsets=100, max_subset_size=1000, ...)`, `prepare`, `feed`,
`summary` -> (fid, fid_mean, fid_cov, kid)) on mmgen's `FID` base [mmgen-memory]: `feed(batch, mode)` extracts features, ALL-GATHERS them
across ranks (lib/apis/test.py:41-53 is the caller; this is the only collective of the eval path) and keeps at most `num_images` rows.

What differs: features stay on the device, the statistics are computed there in float64 (mean / covariance as one GEMM, the matrix square
root of the Frechet distance from a symmetric eigendecomposition, KID as batched GEMMs over all subsets at once), and the feature extractor
is either a plug-in callable `feature_fn` (any [n,3,h,w] float in [-1, 1] -> [n, D] tensor) or, by default, the package's native
Inception-v3 (ssdnerf_b200.inception) loaded at the first `feed` from the StyleGAN TorchScript named by
`inception_args=dict(type='StyleGAN', inception_path=...)`, an external asset that is never downloaded."""
import os
import pickle

import numpy as np
import torch
import torch.distributed as dist

from . import _lib as N
from .registry import Registry

METRICS = Registry('metrics')


def ssim(pred, target):
    """per-image SSIM [n] fp32 of channels-last fp32 pred, target [n, h, w, 3] in [0, 1] on the current CUDA device: the reference's
    `skimage.metrics.structural_similarity(p, t, channel_axis=0, data_range=1)` (lib/core/evaluation/metrics.py:58-71; 7 x 7 uniform
    window, sample covariance) in one launch (csrc/eval_metrics.cu), with fp64 moments.  h, w >= 7."""
    N.require_cuda(pred, target)
    if pred.shape != target.shape or pred.dim() != 4 or pred.shape[-1] != 3:
        raise ValueError(f'ssim: pred and target must both be [n, h, w, 3], got {tuple(pred.shape)} and {tuple(target.shape)}')
    pred, target = pred.float().contiguous(), target.float().contiguous()
    n, h, w, _ = pred.shape
    out = torch.empty(n, dtype=torch.float32, device=pred.device)
    N.check(N.lib().ssdnerf_ssim_f32(N.ptr(pred), N.ptr(target), N.c_u32(n), N.c_u32(h), N.c_u32(w), N.ptr(out), N.stream_ptr()))
    return out


def frechet_distance(mean1, cov1, mean2, cov2):
    """||m1 - m2||^2 + tr(c1) + tr(c2) - 2 tr((c1 c2)^(1/2)) -> (fid, mean term, cov term); float64 tensors.
    tr sqrt(c1 c2) = sum sqrt(eig(c1^(1/2) c2 c1^(1/2))): two symmetric eigendecompositions instead of scipy's Schur-based sqrtm."""
    mean1, mean2, cov1, cov2 = (t.double() for t in (mean1, mean2, cov1, cov2))
    w1, v1 = torch.linalg.eigh(cov1)
    s1 = (v1 * w1.clamp_min(0).sqrt()) @ v1.T
    w = torch.linalg.eigvalsh(s1 @ cov2 @ s1)
    mean_term = (mean1 - mean2).square().sum()
    cov_term = cov1.trace() + cov2.trace() - 2 * w.clamp_min(0).sqrt().sum()
    return float(mean_term + cov_term), float(mean_term), float(cov_term)


def kernel_inception_distance(real_feat, fake_feat, num_subsets=100, max_subset_size=1000, generator=None):
    """metrics.py:160-184 (StyleGAN2-ADA estimator, cubic polynomial kernel), all subsets as one batched GEMM; float64 tensors.
    Subsets are drawn without replacement from `generator` (torch) instead of the global NumPy RNG."""
    real_feat, fake_feat = real_feat.double(), fake_feat.double()
    n = real_feat.shape[1]
    m = min(real_feat.shape[0], fake_feat.shape[0], max_subset_size)
    dev = real_feat.device
    ix = torch.stack([torch.randperm(fake_feat.shape[0], generator=generator)[:m] for _ in range(num_subsets)]).to(dev)
    iy = torch.stack([torch.randperm(real_feat.shape[0], generator=generator)[:m] for _ in range(num_subsets)]).to(dev)
    x, y = fake_feat[ix], real_feat[iy]                                     # [S, m, n]
    a = (x @ x.transpose(1, 2) / n + 1) ** 3 + (y @ y.transpose(1, 2) / n + 1) ** 3
    b = (x @ y.transpose(1, 2) / n + 1) ** 3
    t = (a.sum(dim=(1, 2)) - a.diagonal(dim1=1, dim2=2).sum(dim=1)) / (m - 1) - b.sum(dim=(1, 2)) * 2 / m
    return float(t.sum() / num_subsets / m)


def feature_statistics(feats):
    """mean [D] and unbiased covariance [D, D] (np.cov(rowvar=False)) of feats [n, D] in float64 on the features' device"""
    f = feats.double()
    mean = f.mean(dim=0)
    c = f - mean
    return mean, c.T @ c / (f.shape[0] - 1)


@METRICS.register_module()
class FIDKID:
    name = 'FIDKID'

    def __init__(self, num_images, num_subsets=100, max_subset_size=1000, feature_fn=None, inception_pkl=None, inception_args=None,
                 bgr2rgb=False, image_shape=None):
        self.num_images, self.num_subsets, self.max_subset_size = num_images, num_subsets, max_subset_size
        self.feature_fn, self.inception_pkl, self.bgr2rgb = feature_fn, inception_pkl, bgr2rgb
        self.inception_args = dict(inception_args) if inception_args else None
        self.real_feats, self.fake_feats = [], []
        self.num_real_feeded = self.num_fake_feeded = 0
        self.real_mean = self.real_cov = self.real_feats_all = None
        self._result_dict = {}

    @property
    def num_real_need(self):
        return max(self.num_images - self.num_real_feeded, 0)

    @property
    def num_fake_need(self):
        return max(self.num_images - self.num_fake_feeded, 0)

    def prepare(self):
        """metrics.py:147-158: reference statistics from `tools/inception_stat.py`'s pickle (mean, cov, feats_np)"""
        if self.inception_pkl is not None:
            with open(self.inception_pkl, 'rb') as f:
                ref = pickle.load(f)
            self.real_mean, self.real_cov = torch.as_tensor(ref['mean']).double(), torch.as_tensor(ref['cov']).double()
            self.real_feats_all = torch.as_tensor(ref['feats_np'])
            self.num_real_feeded = self.num_images

    def _native_extractor(self):
        """the package's Inception-v3 (ssdnerf_b200.inception) with the weights of `inception_args['inception_path']`, loaded on first
        use; the file is never downloaded"""
        args = self.inception_args
        if not args:
            raise RuntimeError('FIDKID needs `feature_fn` or `inception_args=dict(type=\'StyleGAN\', inception_path=...)`')
        if args.get('type') != 'StyleGAN':
            raise NotImplementedError(f'FIDKID: inception_args type {args.get("type")!r} is not supported (only \'StyleGAN\')')
        path = args.get('inception_path')
        if not path or not os.path.isfile(path):
            raise RuntimeError(f'FIDKID: the Inception-v3 TorchScript {path!r} was not found (it is an external asset and is never '
                               'downloaded; pass `feature_fn` or place the file there)')
        from .inception import InceptionV3
        return InceptionV3.load(path)

    def feed(self, batch, mode):
        """batch [n,3,h,w] in [-1, 1] -> features -> all-gather over the default process group -> keep what is still needed.
        Returns the number of rows kept (mmgen FID.feed contract [mmgen-memory])."""
        assert mode in ('reals', 'fakes')
        need = self.num_real_need if mode == 'reals' else self.num_fake_need
        if need <= 0:
            return 0
        if self.feature_fn is None:
            self.feature_fn = self._native_extractor()
        if self.bgr2rgb:
            batch = batch[:, [2, 1, 0]]
        with torch.no_grad():
            feat = self.feature_fn(batch).float().contiguous()
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            out = feat.new_empty(dist.get_world_size() * feat.shape[0], feat.shape[1])
            dist.all_gather_into_tensor(out, feat)
            feat = out
        feat = feat[:need]
        if mode == 'reals':
            self.real_feats.append(feat); self.num_real_feeded += feat.shape[0]
        else:
            self.fake_feats.append(feat); self.num_fake_feeded += feat.shape[0]
        return feat.shape[0]

    def _fid(self):
        """(first `num_images` fake features, fid, mean term, cov term); real statistics from the fed reals unless `prepare` loaded them"""
        if self.real_feats_all is None:
            feats = torch.cat(self.real_feats, dim=0)
            assert feats.shape[0] >= self.num_images
            self.real_feats_all = feats[:self.num_images]
            self.real_mean, self.real_cov = feature_statistics(self.real_feats_all)
        fake = torch.cat(self.fake_feats, dim=0)
        assert fake.shape[0] >= self.num_images
        fake = fake[:self.num_images]
        dev = fake.device
        fmean, fcov = feature_statistics(fake)
        return (fake,) + frechet_distance(fmean, fcov, self.real_mean.to(dev), self.real_cov.to(dev))

    @torch.no_grad()
    def summary(self, generator=None):
        fake, fid, mean, cov = self._fid()
        kid = kernel_inception_distance(self.real_feats_all.to(fake.device), fake, self.num_subsets, self.max_subset_size, generator) * 1000
        self._result_dict = dict(fid=fid, fid_mean=mean, fid_cov=cov, kid=kid)
        self._result_str = f'{fid:.4f} ({mean:.5f}/{cov:.5f}), {kid:.4f}'
        return fid, mean, cov, kid


@METRICS.register_module()
class FID(FIDKID):
    """mmgen's `FID` [mmgen-memory], the metric 17 of the 24 shipped configs name: FIDKID's features and Frechet distance without KID.
    `bgr2rgb` defaults to True there (every shipped config sets it to False)."""
    name = 'FID'

    def __init__(self, num_images, image_shape=None, inception_pkl=None, bgr2rgb=True, inception_args=None, feature_fn=None):
        super().__init__(num_images, feature_fn=feature_fn, inception_pkl=inception_pkl, inception_args=inception_args, bgr2rgb=bgr2rgb,
                         image_shape=image_shape)

    @torch.no_grad()
    def summary(self):
        _, fid, mean, cov = self._fid()
        self._result_dict = dict(fid=fid, fid_mean=mean, fid_cov=cov)
        self._result_str = f'{fid:.4f} ({mean:.5f}/{cov:.5f})'
        return fid, mean, cov
