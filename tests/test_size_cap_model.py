"""The independent model of tests/h264_model_size_cap.py names exactly the pictures the oracle recoded and their QP': from the
stream coded with the flag and cap 0 (byte-identical to the flag-off stream) it takes every P picture's count from the syntax reader
alone and applies the rule; the oracle's states with the cap agree up to the first recode (after it the references differ).  A
recoded picture keeps the vectors and reference indices of the flag-off picture wherever both code a P_L0_16x16 macroblock; the
long-term reference is one of the options, so the reader takes ref_idx_l0 from pictures with two active references."""
import pytest

import oracle
from tests import h264_model_size_cap as M
from tests import h264_syntax_refs as HSR
from tests.test_size_cap_oracle import CONTENTS, _encode


@pytest.fixture(scope="module", autouse=True)
def _threads():
    oracle.set_threads(0)


@pytest.mark.parametrize("name", list(CONTENTS))
@pytest.mark.parametrize("qp", [22, 30])
@pytest.mark.parametrize("opts", [dict(), dict(wide=True), dict(droppable=True), dict(ltr=True)])
def test_model_names_the_recoded_pictures(name, qp, opts):
    frames = CONTENTS[name](320, 192)
    zero_aus, _, zero = _encode(frames, 0, qp=qp, **opts)
    model0 = M.decisions(zero_aus, 0)
    for k, (s, d) in enumerate(zip(zero, model0)):
        assert (d is None) == (k == 0), k
        if d is not None:
            assert d[0] == s["bits"] and d[1] == s["qp"], (k, d, s)
    sizes = sorted(-(-d[0] // 8) for d in model0 if d)
    cap = max(1, sizes[-1] // 2)
    model = M.decisions(zero_aus, cap)
    aus, _, st = _encode(frames, cap, qp=qp, **opts)
    first = next(k for k, s in enumerate(st) if s["recoded"])
    assert all(d is None or d[2] == d[1] for d in model[:first])
    assert model[first] is not None and model[first][2] == st[first]["qp_final"]
    a, b = HSR.parse_stream(zero_aus)[first], HSR.parse_stream(aus)[first]
    assert b.qp == st[first]["qp_final"]
    for addr, (x, y) in enumerate(zip(M.vectors(a), M.vectors(b))):
        if x is not None and y is not None:
            assert x == y, (first, addr)      # the vector and ref_idx_l0 the analysis chose
