"""Deterministic, name-keyed fill of BatchNorm running statistics, the companion of param_fill.fill_by_name (which
leaves running_mean / running_var alone): the golden generator (reference model, CPU) and the tests (our model)
give eval-mode BatchNorm identical, non-trivial statistics without storing them."""
import zlib

import torch


@torch.no_grad()
def fill_running_stats_by_name(module: torch.nn.Module, seed: int = 0) -> None:
    """running_mean ~ 0.1 r, running_var = exp(0.2 r) > 0, r ~ N(0, 1) seeded by the buffer's name."""
    for name, t in sorted(module.named_buffers()):
        if not name.endswith(("running_mean", "running_var")):
            continue
        g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(name.encode()))
        r = torch.randn(t.shape, generator=g, dtype=torch.float32)
        v = 0.1 * r if name.endswith("running_mean") else torch.exp(0.2 * r)
        t.copy_(v.to(t.dtype))
