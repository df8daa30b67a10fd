"""Direct FID statistics from finished samples (SURVEY section 8(f)1): the sampler's images go to the feature extractor in
memory and the Inception statistics are accumulated and reduced across ranks, instead of the reference's PNG round trip
(sample.py:312-316 writes files, fid.py:42-71 reads them back).

Reference arithmetic kept verbatim (fid.py:61-79): per rank  mu += f.sum(0);  sigma += f.T @ f  in float64, one all_reduce of
each (NCCL over NVLink on GPUs, gloo in the CPU tests), then  mu /= N;  sigma -= N * mu mu^T;  sigma /= N - 1;
FID = |mu - mu_ref|^2 + tr(sigma + sigma_ref - 2 sqrtm(sigma sigma_ref))  (fid.py:83-87).

The feature extractor itself is the reference's pickled Inception-v3 (`detector_net(images, return_features=True)`, fid.py:34-38,
fetched from a URL): it is a caller-supplied callable here — any `[B,3,H,W] uint8 -> [B,D]` function.
"""
import numpy as np
import torch
import torch.distributed as dist


class FeatureStats:
    """Running first / second moments of feature rows, float64, on the device of the first batch."""

    def __init__(self, feature_dim=None, device=None):
        self.n = 0
        self.mu = None
        self.sigma = None
        if feature_dim is not None:
            self._alloc(feature_dim, device or 'cpu')

    def _alloc(self, d, device):
        self.mu = torch.zeros([d], dtype=torch.float64, device=device)
        self.sigma = torch.zeros([d, d], dtype=torch.float64, device=device)

    def append(self, features):
        """features: [B, D] (any float dtype).  fid.py:69-71."""
        if features.shape[0] == 0:
            return self
        f = features.to(torch.float64)
        if self.mu is None:
            self._alloc(f.shape[1], f.device)
        self.mu += f.sum(0)
        self.sigma += f.T @ f
        self.n += f.shape[0]
        return self

    def append_images(self, images_u8_nhwc, detector):
        """images: [B,H,W,C] uint8 (what dist_utils.to_uint8_nhwc returns / sample.py:311 writes to PNG).  Grey images are
        repeated to 3 channels like fid.py:67-68; the detector receives NCHW uint8 like the reference's data loader yields."""
        x = images_u8_nhwc.permute(0, 3, 1, 2)
        if x.shape[1] == 1:
            x = x.repeat([1, 3, 1, 1])
        return self.append(detector(x))

    def reduce(self):
        """Grand totals over all ranks (fid.py:74-75 + the image count).  No-op without an initialised process group."""
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            n = torch.tensor([float(self.n)], dtype=torch.float64, device=self.mu.device)
            dist.all_reduce(self.mu)
            dist.all_reduce(self.sigma)
            dist.all_reduce(n)
            self.n = int(n.item())
        return self

    def finalize(self):
        """(mu, sigma) as float64 numpy arrays, fid.py:76-79.  Call after reduce()."""
        if self.n < 2:
            raise ValueError(f'need at least 2 images to compute statistics, got {self.n}')     # fid.py:47-48
        mu = self.mu / self.n
        sigma = self.sigma - mu.ger(mu) * self.n
        sigma = sigma / (self.n - 1)
        return mu.cpu().numpy(), sigma.cpu().numpy()


class ScoreStats:
    """Running sum and count of per-image scores (the CLIP score, clip_score.py:89-93: per rank `avg += score.sum()`, then / N over
    all images), float64, with the same all-reduce as FeatureStats."""

    def __init__(self):
        self.total = None
        self.n = 0

    def append(self, scores):
        """scores: [B] per-image scores (B200OpenCLIP.score)."""
        s = scores.to(torch.float64).sum()
        self.total = s if self.total is None else self.total + s
        self.n += scores.shape[0]
        return self

    def reduce(self):
        """Grand totals over all ranks.  No-op without an initialised process group."""
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dev = self.total.device if self.total is not None else ('cuda' if dist.get_backend() == 'nccl' else 'cpu')
            t = torch.stack([torch.as_tensor(0.0 if self.total is None else self.total, dtype=torch.float64, device=dev),
                             torch.tensor(float(self.n), dtype=torch.float64, device=dev)])
            dist.all_reduce(t)
            self.total, self.n = t[0], int(t[1].item())
        return self

    def mean(self):
        """The mean score over every image appended (on all ranks, after reduce())."""
        if self.n < 1:
            raise ValueError('no scores appended')
        return float(self.total) / self.n


def frechet_distance(mu, sigma, mu_ref, sigma_ref):
    """fid.py:83-87 calculate_fid_from_inception_stats."""
    import scipy.linalg
    m = np.square(mu - mu_ref).sum()
    prod = np.dot(sigma, sigma_ref)
    try:
        s, _ = scipy.linalg.sqrtm(prod, disp=False)          # the reference's call; `disp` was removed in recent SciPy
    except TypeError:
        s = scipy.linalg.sqrtm(prod)
    return float(np.real(m + np.trace(sigma + sigma_ref - s * 2)))
