"""CPU: the oracle against the fixtures oracle/make_golden_geometries.py generated from the UNMODIFIED reference at the
geometries the reference builds besides 263 x 196: KIT (251), drop_redundant (67) and AMASS (764) widths, 57 to 224
frames, the transformer's 8-layer MDM and the AdaGN MDM_UNET with keyframe input conditioning.  Same tolerances as
tests/test_oracle_golden.py."""
import pytest
import torch

from oracle import make_golden_geometries as G
from oracle.golden_io import load_golden


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "geometries")


def test_fixture_holds_every_case(gold):
    want = {f"{n}.{k}.{i}" for n, c in G.CASES.items() for k in ("fwd", "tail") + (("fwd_cfg",) if c.get("text") else ())
            for i in range(G.B)}
    assert set(gold) == want
    for n, c in G.CASES.items():
        assert G.fixture(gold, f"{n}.fwd").shape == (G.B, c["D"], 1, c["L"])


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_reproduces_the_reference_at_this_geometry(gold, name):
    gi = G.case_inputs(name)
    mask = gi["mask"].double().mean().item()
    assert 0.1 < mask < 0.3, mask          # about 20 % observed, as the fixtures were made
    got = G.oracle_outputs(name)
    for key, value in got.items():
        rtol, atol = G.tolerance(name, key)
        want = torch.from_numpy(G.fixture(gold, f"{name}.{key}"))
        err = (value - want).abs().max().item()
        assert torch.allclose(value, want, rtol=rtol, atol=atol), (key, err)
