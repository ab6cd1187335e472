"""The flagship transformer pass runs the chained layer kernel, not the one-launch-per-layer fallback.

The engine falls back to the unchained path when fewer than num_sms / 2 CTA pairs of linear_chain_kernel can be
resident at once. That fallback computes the same samples, only slower, so nothing else would notice it: here one
profiled pass at B = 64 must show a chained launch per encoder layer, at bf16x3 and at bf16.
"""
import pytest
import torch

import condmdi_b200 as C

pytestmark = pytest.mark.gpu

LAYERS = 8


@pytest.mark.parametrize("precision", [C.capi.PRECISION_BF16X3, C.capi.PRECISION_BF16], ids=["bf16x3", "bf16"])
def test_profile_pass_is_chained(precision):
    torch.manual_seed(0)
    m = C.MDM(njoints=263, nfeats=1, latent_dim=512, ff_size=1024, num_layers=LAYERS, num_heads=4, cond_mode="no_cond").cuda()
    eng = m.engine_for(torch.device("cuda", 0), max_batch=64, precision=precision)
    names = [n for n, _ in eng.profile_pass(64, repeats=1)]
    chained = [n for n in names if n in ("chain", "chain_last")]
    assert len(chained) == LAYERS, names
    assert all(ms > 0 for _, ms in eng.profile_pass(64, repeats=1))
