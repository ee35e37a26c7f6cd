"""Writes the 2^(i/n) tables of the reduced-range exps (kg_mc.cuh, cov.cu) as C hexadecimal double literals, one per
line, each the correctly rounded value:

    python cornell-moe_b200/csrc/make_exp2_table.py 64   > cornell-moe_b200/csrc/exp2_table64.inc
    python cornell-moe_b200/csrc/make_exp2_table.py 2048 > cornell-moe_b200/csrc/exp2_table2048.inc

The values come from mpmath at 200 bits where it is installed, else from `fractions`: the largest double x <= 2^(i/n)
found by bisection on x^n <= 2^i in exact rational arithmetic, then rounded to nearest by comparing the midpoint."""
import sys
from fractions import Fraction


def exp2_frac(i, n):
    """2^(i/n), 0 <= i < n, correctly rounded to double with exact arithmetic only."""
    # doubles in [1, 2) are m / 2^52 with 2^52 <= m < 2^53; find the largest m with (m / 2^52)^n <= 2^i
    lo, hi = 1 << 52, 1 << 53
    target = Fraction(2) ** i
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if Fraction(mid, 1 << 52) ** n <= target:
            lo = mid
        else:
            hi = mid
    # round to nearest: the true value lies in [lo, lo + 1) ulps; it is never exactly a midpoint (2^(i/n) is irrational
    # for 0 < i < n), so comparing the midpoint's n-th power decides
    if i and Fraction(2 * lo + 1, 1 << 53) ** n <= target:
        lo += 1
    return float(Fraction(lo, 1 << 52))


def exp2_mp(i, n):
    import mpmath as mp
    mp.mp.prec = 200
    return float(mp.power(2, mp.mpf(i) / n))


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    try:
        import mpmath  # noqa: F401
        f = exp2_mp
    except ImportError:
        f = exp2_frac
    for i in range(n):
        print(f"{float.hex(f(i, n))},")


if __name__ == "__main__":
    main()
