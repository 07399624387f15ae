"""Latent-strand test infrastructure: a small deterministic stand-in for the strand networks of
GaussianModelHair (reference src/scene/gaussian_model_latent_strands.py), whose outputs reach the model by the
expressions of its generate_strands() (:442-484).  Its cost is not the reference networks' cost."""
from __future__ import annotations

import torch
from torch import nn

import _util

synth = _util.synth


def polyline(hair_scene, S: int) -> torch.Tensor:
    """(S, L+1, 3) polyline points whose midpoints and segment vectors are the strand scene's `xyz` and `dir`
    (oracle/synth.py make_strand_scene)."""
    d = hair_scene["dir"].view(S, -1, 3)
    p0 = hair_scene["xyz"].view(S, -1, 3)[:, :1] - 0.5 * d[:, :1]
    return torch.cat([p0, p0 + torch.cumsum(d, dim=1)], dim=1)


class StandInDecoder(nn.Module):
    """Trainable polyline points `p` (S, L+1, 3) and a per-segment appearance latent through a linear colour decoder.
    generate(hair) sets `_xyz`, `_dir`, `_features_dc`, `_features_rest` and `_orient_conf` on `hair` the way
    generate_strands() does and returns a diffusion dict with a stand-in prior term "L_diff"."""

    def __init__(self, S: int, L: int, seed: int):
        super().__init__()
        scene = synth.make_strand_scene(S, seed=seed, segments=L)
        self.p = nn.Parameter(polyline(scene, S))
        g = torch.Generator().manual_seed(seed + 1)
        self.z = nn.Parameter(0.5 * torch.randn(S, L, 16, generator=g))
        self.color = nn.Linear(16, 3 + 45 + 1)
        with torch.no_grad():
            self.color.weight.copy_(0.3 * torch.randn(49, 16, generator=g))
            self.color.bias.copy_(0.1 * torch.randn(49, generator=g))

    def generate(self, hair) -> dict:
        p = self.p
        S, L = p.shape[0], p.shape[1] - 1
        hair._xyz = (p[:, 1:] + p[:, :-1]).view(-1, 3) * 0.5
        hair._dir = (p[:, 1:] - p[:, :-1]).view(-1, 3)
        f_dc, f_rest, conf = self.color(self.z).split([3, 45, 1], dim=-1)
        hair._features_dc = f_dc.reshape(S * L, 1, 3)
        hair._features_rest = f_rest.reshape(S * L, 15, 3)
        hair._orient_conf = conf.reshape(S * L, 1)
        return {"L_diff": (hair._dir.norm(dim=-1) - 0.002).square().mean() * 1e4}
