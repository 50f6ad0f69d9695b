"""ViT workload. The reference's script (/root/reference/models/vit/train_vit.py:30-63) trains
``vit_pytorch.ViT(image_size=256, patch_size=32, dim=1024, depth=6, heads=16, mlp_dim=2048)`` on
synthetic batches of 256 images under plain DDP; BASELINE.json names ViT-B/16 for the H100 config
("ViT-B/16 DDP with reconstruct_topology every 500 steps"). Both shapes are available here; the
model is a standard pre-norm ViT on ``scaled_dot_product_attention``."""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn as nn
import torch.nn.functional as F


@dataclass
class ViTConfig:
    """The reference's ViT workload shape (``vit_pytorch.ViT(image 256, patch 32, dim 1024, depth 6, heads 16, mlp
    2048)``, /root/reference/models/vit/train_vit.py:30-40)."""

    image_size: int = 224
    patch_size: int = 16
    dim: int = 768
    depth: int = 12
    heads: int = 12
    mlp_dim: int = 3072
    num_classes: int = 1000
    channels: int = 3

    @classmethod
    def b16(cls):                       # BASELINE.json config 4
        return cls()

    @classmethod
    def reference(cls):                 # models/vit/train_vit.py:30-40
        return cls(image_size=256, patch_size=32, dim=1024, depth=6, heads=16, mlp_dim=2048)

    @classmethod
    def tiny(cls):
        return cls(image_size=32, patch_size=8, dim=64, depth=2, heads=4, mlp_dim=128, num_classes=10)


class _Block(nn.Module):
    def __init__(self, c: ViTConfig):
        super().__init__()
        self.heads = c.heads
        self.ln1, self.ln2 = nn.LayerNorm(c.dim), nn.LayerNorm(c.dim)
        self.qkv, self.proj = nn.Linear(c.dim, 3 * c.dim), nn.Linear(c.dim, c.dim)
        self.fc1, self.fc2 = nn.Linear(c.dim, c.mlp_dim), nn.Linear(c.mlp_dim, c.dim)

    def forward(self, x):
        B, N, D = x.shape
        q, k, v = self.qkv(self.ln1(x)).view(B, N, 3, self.heads, D // self.heads).permute(2, 0, 3, 1, 4)
        x = x + self.proj(F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, N, D))
        return x + self.fc2(F.gelu(self.fc1(self.ln2(x))))


class ViT(nn.Module):
    """Vision transformer classifier (patch embedding by a strided conv, pre-LN blocks with SDPA attention, class
    token) — self-contained so the workload does not need ``vit_pytorch``."""

    def __init__(self, c: ViTConfig = None):
        super().__init__()
        self.cfg = c = c or ViTConfig()
        n = (c.image_size // c.patch_size) ** 2
        self.patch = nn.Conv2d(c.channels, c.dim, c.patch_size, c.patch_size)
        self.cls = nn.Parameter(torch.zeros(1, 1, c.dim))
        self.pos = nn.Parameter(torch.randn(1, n + 1, c.dim) * 0.02)
        self.blocks = nn.ModuleList([_Block(c) for _ in range(c.depth)])
        self.norm = nn.LayerNorm(c.dim)
        self.head = nn.Linear(c.dim, c.num_classes)

    def forward(self, images, labels=None):
        x = self.patch(images).flatten(2).transpose(1, 2)
        x = torch.cat([self.cls.expand(x.shape[0], -1, -1).to(x.dtype), x], 1) + self.pos.to(x.dtype)
        for b in self.blocks:
            x = b(x)
        logits = self.head(self.norm(x[:, 0]))
        if labels is None:
            return logits
        return F.cross_entropy(logits.float(), labels), logits
