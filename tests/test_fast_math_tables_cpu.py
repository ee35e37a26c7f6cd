"""The 2^(i/n) tables of the reduced-range exps (exp_tab, exp_tab_cov: 64 entries; exp_tab2k: 2048 entries).

Every entry must be 2^(i/n) correctly rounded to double, checked with make_exp2_table.py's exact rational method (no
floating point anywhere); the generator must reproduce both committed files byte for byte; and the 64-entry table must
be every 32nd entry of the 2048-entry one, so that exp_tab and exp_tab2k agree at the shared nodes."""
import importlib.util
import os
import subprocess
import sys
from fractions import Fraction

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cornell-moe_b200", "csrc")


def _gen():
    spec = importlib.util.spec_from_file_location("make_exp2_table", os.path.join(CSRC, "make_exp2_table.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _table(n):
    with open(os.path.join(CSRC, f"exp2_table{n}.inc")) as f:
        lines = f.read().splitlines()
    assert len(lines) == n and all(s.endswith(",") for s in lines)
    return [float.fromhex(s[:-1]) for s in lines]


def _correctly_rounded(x, i, n):
    """x is the double nearest 2^(i/n): x^n and its neighbours' midpoints' n-th powers bracket 2^i exactly."""
    target = Fraction(2) ** i
    fx = Fraction(x)
    ulp = Fraction(1, 1 << 52)  # every entry lies in [1, 2)
    if not 1 <= fx < 2:
        return False
    if i == 0:
        return fx == 1
    lo, hi = fx - ulp / 2, fx + ulp / 2
    # 2^(i/n) is irrational for 0 < i < n, so it is never a midpoint: strict brackets
    return lo ** n < target < hi ** n


@pytest.mark.parametrize("n", [64, 2048])
def test_every_entry_correctly_rounded(n):
    tab = _table(n)
    bad = [i for i, x in enumerate(tab) if not _correctly_rounded(x, i, n)]
    assert not bad, f"exp2_table{n}.inc entries not correctly rounded: {bad[:10]}"


@pytest.mark.parametrize("n", [64, 2048])
def test_generator_reproduces_file(n):
    out = subprocess.run([sys.executable, os.path.join(CSRC, "make_exp2_table.py"), str(n)], check=True,
                         capture_output=True).stdout
    with open(os.path.join(CSRC, f"exp2_table{n}.inc"), "rb") as f:
        assert out == f.read()


def test_generator_exact_method_matches_file():
    """The generator's mpmath-free path (exact rationals) gives the committed 64-entry table and a sample of the 2048."""
    gen = _gen()
    assert [gen.exp2_frac(i, 64) for i in range(64)] == _table(64)
    t2k = _table(2048)
    for i in list(range(0, 2048, 97)) + [1, 2047]:
        assert gen.exp2_frac(i, 2048) == t2k[i], i


def test_small_table_is_every_32nd_entry():
    assert _table(64) == _table(2048)[::32]
