"""Every case of the fp16/bf16 convolution case table (tests/conv_cases.py) on the H100, against an fp64 convolution of
the same rounded operands: |got - ref| <= ulp_out(|ref|) + tau(K) * (conv(|x|, |w|) + |b| (+ |res|)).  Each case also
checks the channel sentinels and the guard image after the view, that a second launch gives the same bits, and that a
two-CTA launch writes the bits of the one-CTA launch (reserved bit 4).  Run with -s for the worst fraction of the bound
per case."""
import pytest

from conv_cases import CASES, check_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", CASES, ids=[c.name.replace(" ", "_") for c in CASES])
def test_conv_case_against_fp64(case):
    check_case(case)
