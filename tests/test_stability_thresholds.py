"""The stability screen's decision boundaries on the CPU: the boundary pairs and molecules of oracle/stability_cases.py are what they
claim to be (checked with exact rational arithmetic), the builder is deterministic and covers every threshold of the reference's
tables, and `restate.check_stability` equals the unmodified reference on all of them (tests/golden/reference_pins_stability_thresholds.pt,
made by oracle/make_stability_pins.py).  tests/test_gpu_stability.py runs the device screen on the same inputs."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import make_stability_pins as msp, restate, stability_cases as sc


@pytest.fixture(scope='module')
def pins():
    return torch.load(msp.OUT, weights_only=True)


def _exact_round(q):
    return float(q)                     # Fraction -> nearest double, ties to even


def test_thresholds_are_the_reference_tables():
    th = sc.thresholds()
    assert len(th) == 36 + 9 + 4 + 2
    assert len({(o, e1, e2) for o, e1, e2, _ in th[:-2]}) == len(th) - 2
    doubles = {(sc.ELEMENTS[e1], sc.ELEMENTS[e2]) for o, e1, e2, _ in th if o == 2 and e1 + e2 > 0}
    assert doubles == {('C', 'C'), ('C', 'N'), ('C', 'O'), ('C', 'S'), ('N', 'N'), ('N', 'O'), ('O', 'O'), ('O', 'P'), ('P', 'S')}
    triples = {(sc.ELEMENTS[e1], sc.ELEMENTS[e2]) for o, e1, e2, _ in th if o == 3 and e1 + e2 > 0}
    assert triples == {('C', 'C'), ('C', 'N'), ('C', 'O'), ('N', 'N')}
    assert th[-2:] == [(2, 0, 0, 4), (3, 0, 0, 2)]
    for o, e1, e2, T in th:                                             # the pair gains order o at T, and no other order does
        assert restate.get_bond_order(e1, e2, (T - 0.5) / 100) >= o and restate.get_bond_order(e1, e2, (T + 0.5) / 100) == o - 1


def test_reachable_values_with_exact_arithmetic():
    """For every threshold, the values fl(100 * y) of all doubles y whose product lies within three ulps of T: T itself is among them
    unless T is 111, 113, 116 or 220, and sc.reachable names the nearest ones on each side."""
    no_eq = []
    for _, _, _, T in sc.thresholds():
        ulp = math.ulp(float(T))
        y = float(T) / 100
        while Fraction(100) * Fraction(y) > T - 3 * ulp:
            y = math.nextafter(y, 0)
        vals = set()
        while Fraction(100) * Fraction(y) < T + 3 * ulp:
            vals.add(_exact_round(Fraction(100) * Fraction(y)))
            y = math.nextafter(y, math.inf)
        eq, lo, hi = sc.reachable(T)
        assert (T in vals) == (eq is not None), T
        assert lo == max(v for v in vals if v < T) and hi == min(v for v in vals if v > T), T
        assert T - lo in (ulp, 2 * ulp) and hi - T in (ulp, 2 * ulp) or T <= 4, T
        if eq is None:
            no_eq.append(T)
    assert sorted(set(no_eq)) == [111, 113, 116, 220]


def test_every_case_is_what_it_claims():
    """'eq' / 'below' / 'above': the reference's expression gives T / its nearest values; 'fma': the exact products and sums of both
    contraction orders, each rounded once, put the pair on the other side of T.  Every coordinate is an fp32 value."""
    cases = sc.pair_cases()
    fma_sides = set()
    for c in cases:
        p1, p2, T = c['p1'], c['p2'], c['T']
        for p in (p1, p2):
            assert np.array_equal(p.astype(np.float32).astype(np.float64), p)
        d = sc.reference_distance(p1, p2)
        if c['kind'] == 'coincident':
            assert d == 0 and restate.get_bond_order(c['e1'], c['e2'], d / 100) == 3
            continue
        eq, lo, hi = sc.reachable(T)
        want = {'eq': eq, 'below': lo, 'above': hi}.get(c['kind'])
        if want is not None:
            assert d == want, (sc.case_name(c), d)
        else:
            dx, dy, dz = (Fraction(float(v)) for v in (p1 - p2))
            for first, second in ((dx, dy), (dy, dx)):
                s = _exact_round(dz * dz + Fraction(_exact_round(second * second + Fraction(float(first * first)))))
                assert (100 * float(np.sqrt(s)) < T) != (d < T), sc.case_name(c)
            fma_sides.add(d < T)
        order = restate.get_bond_order(c['e1'], c['e2'], np.sqrt(np.sum((p1 - p2) ** 2)))
        assert (order >= c['order']) == (d < T)
    assert fma_sides == {True, False}                                  # contracted forms wrong in both directions


def test_builder_is_deterministic_and_covers_every_threshold(pins):
    cases = sc.pair_cases()
    got = {(c['order'], c['e1'], c['e2'], c['T']): set() for c in cases}
    for c in cases:
        got[c['order'], c['e1'], c['e2'], c['T']].add(c['kind'])
    for o, e1, e2, T in sc.thresholds():
        assert got.pop((o, e1, e2, T)) == set(sc.wanted_kinds(T)), (o, e1, e2, T)
    assert sorted(got.values()) == [{'coincident'}] * 3
    inputs = sc.inputs()
    assert [c['name'] for c in inputs] == pins['names']
    assert torch.equal(torch.from_numpy(np.concatenate([c['pos'] for c in inputs])), pins['pos'])
    assert torch.equal(torch.from_numpy(np.concatenate([c['z'] for c in inputs])), pins['z'])


def test_molecules_hinge_on_the_boundary_pair(pins):
    """The carbon's fourth hydrogen: stable molecule (with and without hs) exactly when the boundary pair is a bond."""
    names = pins['names']
    mols = sc.molecules()
    assert [m['name'] for m in mols] == ['CH4_%s' % k for k in sc.wanted_kinds(119)]
    for m in mols:
        bonded = sc.reference_distance(m['pos'][0], m['pos'][1]) < 119
        r = pins['result'][names.index(m['name'])]
        assert r[:, 0].tolist() == [int(bonded)] * 2, m['name']
        assert r[1, 1] == (5 if bonded else 3), m['name']            # hs: the carbon is stable only at 4 == bonds, the H4 at 1 == 1
    assert {bool(sc.reference_distance(m['pos'][0], m['pos'][1]) < 119) for m in mols} == {True, False}


def test_restatement_equals_reference_pins(pins):
    cuts = np.cumsum([0] + pins['counts'].tolist())
    pos, z = pins['pos'].numpy(), pins['z'].numpy()
    for m, name in enumerate(pins['names']):
        a, b = cuts[m], cuts[m + 1]
        for hs in (False, True):
            w = restate.check_stability(pos[a:b], z[a:b], hs=hs)
            assert [int(w[0]), w[1], w[2]] == pins['result'][m, int(hs)].tolist(), (name, hs)
            assert np.array_equal(w[3], pins['nr_bonds'][a:b, int(hs)].numpy()), (name, hs)
