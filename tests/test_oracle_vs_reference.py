"""Comparison of the oracle port with the reference itself: tests/golden/reference_model.pt holds what the unmodified
reference model computed (oracle/make_golden.py, golden_reference_model) — its state-dict shapes and its outputs on
seeded cases — so the port is pinned against the reference without the reference installed."""
from pathlib import Path

import torch

from oracle import cases as Cs
from oracle.make_golden import state_spec_digest
from oracle import unet_port as P

GOLDEN = Path(__file__).resolve().parent / "golden" / "reference_model.pt"


def _golden():
    return torch.load(GOLDEN, weights_only=False)


def test_reference_state_dict_keys_and_port_output():
    g = _golden()
    case = Cs.GOLDEN_CASES[1]                      # non-2:1 views -> exercises the view-height shim
    assert g["case"] == case.name
    spec = P.state_spec(case.net_config())
    assert len(spec) == g["state_spec_len"] and state_spec_digest(spec) == g["state_spec_sha256"]
    sd = Cs.make_weights(case)
    x, t, c = Cs.make_inputs(case)
    out = P.wrapper_forward(sd, case.net_config(), x, t, c)
    assert (out - g["eps"]).abs().max().item() < 2e-5


def test_fresh_reference_model_outputs_zero():
    """SURVEY.md section 0.3: zero_module'd tails make a fresh model predict exactly 0."""
    g = _golden()
    assert g["fresh_case"] == Cs.GOLDEN_CASES[0].name
    assert g["fresh_max_abs"] == 0.0
