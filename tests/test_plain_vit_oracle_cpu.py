"""The plain-ViT oracle (oracle/plain_vit_oracle.py::forward_fp32 on a vitl16_384 / vitb16_384 state_dict) against the
golden vectors of the UNMODIFIED reference class (oracle/make_golden.py::make_large_golden), at every tap and with the
bound the hybrid restatement meets on its own goldens (tests/test_oracle_cpu.py).  Its float64 evaluation is the
gradient truth of tests/test_plain_vit_train_gpu.py."""
from pathlib import Path

import pytest
import torch

from oracle import make_golden, plain_vit_oracle

GOLDEN = Path(__file__).parent / "golden"
CASES = {"vitl16_384": "dpt_large_fp32_seed0_c1.pt", "vitb16_384": "dpt_vitb16_fp32_seed0_c1.pt"}


@pytest.mark.parametrize("backbone", sorted(CASES))
def test_plain_vit_oracle_matches_reference_golden(backbone, monkeypatch):
    from omnidata_b200.synthetic import make_state_dict
    rec = torch.load(GOLDEN / CASES[backbone])
    sd = make_state_dict(0, 1, spec=[(k, tuple(s)) for k, s in rec["spec"]])
    x = make_golden.golden_input(1)
    taps = {}
    with torch.no_grad():
        y = plain_vit_oracle.forward_fp32(sd, x, taps)
    assert tuple(y.shape) == (1, 384, 384)
    ref = rec["output_sub8"]
    assert float((y[..., ::8, ::8] - ref).norm() / ref.norm()) < 1e-5
    monkeypatch.setattr(make_golden, "N_SAMPLES", len(next(iter(rec["taps"].values()))["samples"]))
    assert len(rec["taps"]) == 13
    for name, g in rec["taps"].items():
        t = taps[name]
        assert list(t.shape) == g["shape"], name
        t = t.reshape(-1)
        s = t[make_golden.sample_indices(t.numel(), name)]
        err = float((s - g["samples"]).norm() / (g["samples"].norm() + 1e-12))
        assert err < 1e-5, f"{name}: {err}"
        assert abs(float(t.pow(2).mean().sqrt()) - g["rms"]) < 1e-4 * max(1.0, g["rms"])
