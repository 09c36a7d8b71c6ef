# -*- coding: utf-8 -*-
"""The bf16 verify path bit for bit against digests recorded on an H100 (tests/golden/gen_verify_bits_golden.py):
the gate_up and lm_head weight-streaming GEMMs at the benchmark's shapes and 1, 17, 63 and 64 rows, and the logits of
the full Llama-2-7B-shape verify forward at P = 384 and P = 3968.  A kernel change that reorders any fp32 sum fails
here even when every tolerance-based test still passes."""
import json

import pytest

from tests.golden import gen_verify_bits_golden as gen

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def golden():
    with open(gen.OUT) as f:
        return json.load(f)


def test_gemm_outputs_match_the_recorded_digests(golden):
    got = gen.gemm_digests()
    bad = [k for k in got if got[k] != golden[k]]
    assert not bad, f'GEMM outputs changed bits: {bad}'


def test_verify_forward_logits_match_the_recorded_digests(golden):
    got = gen.forward_digests()
    bad = [k for k in got if got[k] != golden[k]]
    assert not bad, f'verify-forward logits changed bits: {bad}'
