"""Drop-in for ``ldm.modules.distributions.distributions.DiagonalGaussianDistribution``: the posterior that
``AutoencoderKL.encode`` returns (ldm/models/autoencoder.py:345-349).

Same constructor, attributes (``parameters``, ``mean``, ``logvar`` clamped to [-30, 20], ``std``, ``var``,
``deterministic``) and methods (``sample``, ``mode``, ``kl``, ``nll``) as the reference class
(ldm/modules/distributions/distributions.py:24-59).  ``AutoencoderKLWithEncoder.encode`` uses it only when the
reference class is unknown: ``install(first_stage=True)`` records the reference's own class, because
``LatentDiffusion.get_first_stage_encoding`` (ddpm_audio.py:157-164) checks ``isinstance`` against it.

These are a handful of elementwise ops on the [B, 2*embed_dim, h, w] moments: plumbing, left to PyTorch.
"""
from __future__ import annotations

import math

import torch


class DiagonalGaussianDistribution:
    def __init__(self, parameters, deterministic=False):
        self.parameters = parameters
        mean, logvar = torch.chunk(parameters, 2, dim=1)
        self.mean = mean
        self.logvar = logvar.clamp(-30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if deterministic:
            self.std = torch.zeros_like(self.mean)
            self.var = torch.zeros_like(self.mean)

    def sample(self):
        # the noise is drawn on the host and then moved, so that a seeded run consumes the CPU generator exactly as the
        # reference does
        eps = torch.randn(self.mean.shape).to(device=self.parameters.device)
        return self.mean + self.std * eps

    def mode(self):
        return self.mean

    def kl(self, other=None):
        """KL(self || other), other = N(0, I) by default; summed over [1, 2, 3]."""
        if self.deterministic:
            return torch.Tensor([0.0])
        if other is None:
            terms = self.mean.pow(2) + self.var - 1.0 - self.logvar
        else:
            terms = ((self.mean - other.mean).pow(2) / other.var + self.var / other.var - 1.0 - self.logvar
                     + other.logvar)
        return 0.5 * torch.sum(terms, dim=[1, 2, 3])

    def nll(self, sample, dims=(1, 2, 3)):
        """negative log-likelihood of ``sample``, summed over ``dims``."""
        if self.deterministic:
            return torch.Tensor([0.0])
        return 0.5 * torch.sum(math.log(2.0 * math.pi) + self.logvar + (sample - self.mean).pow(2) / self.var,
                               dim=list(dims))
