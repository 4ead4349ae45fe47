"""calculate_distance (mod.rs:218-231, `orc.haversine_km`) against a 50-digit great-circle distance at the edges of the
coordinate space: the poles, the antimeridian, longitudes outside ±180, exact and near antipodes, identical points
and one place written twice with a latitude beyond ±90.  Proximity groups depend only on the ORDER of distances, and
that order is what goes wrong at these edges; the device haversines restate this function operation by operation.

Why the tolerance is absolute near a = 0 and a = 1.  With a = sin²(Δφ/2) + cos φ₁·cos φ₂·sin²(Δλ/2) the distance is
c = 2·atan2(√a, √(1−a)), and dc/da = 1/√(a·(1−a)).  An absolute error ε in a therefore moves c by at most about
2·√ε where a or 1−a is itself of the order of ε, whatever the distance.  Near an antipode a ≈ 1 is the sum of two terms
of size up to 1, each rounded, so ε is a few units u = 2⁻⁵³ and √(1−a) is computed from cancelled digits: the error is
up to 2·R·√(2u) ≈ 1.9e-4 km for an exact antipode, hence ≤ 2e-4 km within 1 km of one.  Away from the antipode,
1−a ≥ (δ/2R)² for a distance δ short of it and the error falls as u/√(1−a).  For real latitudes a ≈ 0 is a sum of two
non-negative terms with small RELATIVE error, and the distance keeps 1e-9 relative accuracy.  With a latitude beyond
±90, cos φ₁·cos φ₂ < 0 and a is a difference of terms up to 1: the same place written twice comes out within
2·R·√(4u) ≈ 2.7e-4 km of 0 (3u was the largest error over 20 000 random such pairs).
"""
import math

import mpmath
import numpy as np
import pytest

from oracle import pm_oracle as orc

R = 6371.0
RADS_PER_DEG = 3.14159265358979323846264338327950288 / 180.0
U = 2.0 ** -53
HALF_CIRCUMFERENCE_KM = float(mpmath.mpf(R) * mpmath.pi)
ANTIPODE_TOL_KM = 2e-4
CANCEL_TOL_KM = 2.0 * R * math.sqrt(4.0 * U)


def reference_km(lat1, lon1, lat2, lon2) -> float:
    """Great-circle distance from unit vectors: atan2(|p × q|, p · q), well conditioned at antipodes and at 0."""
    with mpmath.workdps(50):
        k = mpmath.pi / 180

        def unit(lat, lon):
            la, lo = mpmath.mpf(lat) * k, mpmath.mpf(lon) * k
            return mpmath.cos(la) * mpmath.cos(lo), mpmath.cos(la) * mpmath.sin(lo), mpmath.sin(la)

        p, q = unit(lat1, lon1), unit(lat2, lon2)
        cross = (p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0])
        dot = p[0] * q[0] + p[1] * q[1] + p[2] * q[2]
        return float(R * mpmath.atan2(mpmath.sqrt(sum(x * x for x in cross)), dot))


def restated_a(lat1, lon1, lat2, lon2) -> float:
    """a as calculate_distance forms it, before the clamp (glibc through CPython's math, as the oracle)."""
    s1 = math.sin((lat2 - lat1) * RADS_PER_DEG / 2.0)
    s2 = math.sin((lon2 - lon1) * RADS_PER_DEG / 2.0)
    return s1 * s1 + math.cos(lat1 * RADS_PER_DEG) * math.cos(lat2 * RADS_PER_DEG) * (s2 * s2)


def tolerance_km(ref, pair) -> float:
    if ref > HALF_CIRCUMFERENCE_KM - 1.0:
        return ANTIPODE_TOL_KM
    if ref < 1.0 and max(abs(pair[0]), abs(pair[2])) > 90.0:
        return CANCEL_TOL_KM
    return 1e-9 * ref + 1e-6


def twice_written(lat, lon):
    """The place (lat, lon), |lat| <= 90, written with its latitude beyond ±90: (±180 − lat, lon + 180)."""
    return (math.copysign(180.0, lat) - lat, lon + 180.0)


def _rng_pairs(seed, n, make):
    rng = np.random.default_rng(seed)
    return [make(rng) for _ in range(n)]


def _metres_north(lat, lon, m):
    return lat + m / 1000.0 / R / RADS_PER_DEG, lon


PLACEMENTS = {
    # both poles: a pole written with different longitudes is one place; pairs across the pole and on one meridian
    "poles": [(90.0, 0.0, 90.0, 123.456), (-90.0, -170.0, -90.0, 10.0), (90.0, 0.0, -90.0, 0.0),
              (89.9999, 17.0, 90.0, -163.0), (89.5, 0.0, 89.5, 180.0), (-89.99, 45.0, -89.99, -135.0),
              (88.0, 33.0, 85.0, 33.0), (-87.5, -120.0, -89.999999, -120.0)]
             + _rng_pairs(11, 300, lambda r: (float(np.copysign(90.0 - r.uniform(0, 3) ** 3, s := r.choice([-1, 1]))),
                                             float(r.uniform(-180, 180)),
                                             float(np.copysign(90.0 - r.uniform(0, 3) ** 3, s)),
                                             float(r.uniform(-180, 180)))),
    # pairs across ±180, in both conventions (179.9 and -180.1 are one meridian)
    "antimeridian": [(10.0, 179.9, 10.0, -179.9), (10.0, 179.9, 10.0, -180.1), (0.0, 180.0, 0.0, -180.0),
                     (-45.0, -180.0, -45.0, 180.0), (60.0, 179.999999, 60.0, -179.999999)]
                    + _rng_pairs(12, 300, lambda r: (float(r.uniform(-89, 89)), float(180.0 - r.uniform(0, 0.5)),
                                                    float(r.uniform(-89, 89)), float(r.uniform(-180.5, -179.5)))),
    # longitudes outside ±180, up to three turns
    "wrapped_longitudes": [(20.0, 540.0, 20.0, 180.0), (-33.0, -721.5, -33.0, -1.5), (5.0, 1000.0, -5.0, -1000.0)]
                          + _rng_pairs(13, 300, lambda r: (float(r.uniform(-90, 90)),
                                                          float(r.uniform(-180, 180) + 360.0 * r.integers(-3, 4)),
                                                          float(r.uniform(-90, 90)),
                                                          float(r.uniform(-180, 180) + 360.0 * r.integers(-3, 4)))),
    # exact antipodes (of the f64 coordinates given) and points metres from them
    "antipodes": [(0.0, 0.0, 0.0, 180.0), (90.0, 0.0, -90.0, 0.0), (45.0, 10.0, -45.0, -170.0),
                  (-76.39166335263677, 48.73755368270059, 76.39166335263677, 48.73755368270059 + 180.0)]
                 + _rng_pairs(14, 2000, lambda r: (la := float(r.uniform(-90, 90)), lo := float(r.uniform(-180, 180)),
                                                  -la, lo + 180.0)),
    "near_antipodes": _rng_pairs(15, 600, lambda r: (la := float(r.uniform(-89, 89)), lo := float(r.uniform(-180, 180)),
                                                    *_metres_north(-la, lo + 180.0, float(r.choice([-1, 1]) * 10.0 ** r.uniform(0, 3))))),
    "identical": [(0.0, 0.0, 0.0, 0.0), (90.0, 0.0, 90.0, 0.0), (-90.0, 180.0, -90.0, 180.0), (12.5, 540.0, 12.5, 540.0)]
                 + _rng_pairs(16, 200, lambda r: (la := float(r.uniform(-90, 90)), lo := float(r.uniform(-180, 180)), la, lo)),
    # one place written twice, once with a latitude beyond ±90 (the clamp below 0)
    "twice_written": [(102.09351324162789, 125.07614529740374, 180.0 - 102.09351324162789, 125.07614529740374 + 180.0)]
                     + _rng_pairs(17, 2000, lambda r: (la := float(r.uniform(-90, 90)), lo := float(r.uniform(-180, 180)),
                                                      *twice_written(la, lo))),
}


@pytest.mark.parametrize("placement", list(PLACEMENTS))
def test_distance_matches_high_precision_reference(placement):
    worst = 0.0
    for pair in PLACEMENTS[placement]:
        d = orc.haversine_km(*pair)
        ref = reference_km(*pair)
        assert not math.isnan(d), f"{pair}: NaN distance (a = {restated_a(*pair)!r})"
        err = abs(d - ref)
        assert err <= tolerance_km(ref, pair), f"{pair}: {d!r} km vs {ref!r} km"
        worst = max(worst, err / tolerance_km(ref, pair))
    print(f"\n[{placement}] worst error / tolerance = {worst:.3f}")


def test_same_point_written_beyond_90_is_at_distance_zero():
    """(φ, λ) and (180 − φ, λ + 180) with φ in (90, 180) are one place; a rounds to −2.8e-17 here, and sqrt(a) used
    to make the distance NaN — which no comparison orders."""
    pair = (102.09351324162789, 125.07614529740374, 180.0 - 102.09351324162789, 125.07614529740374 + 180.0)
    assert restated_a(*pair) < 0.0
    assert orc.haversine_km(*pair) == 0.0
    assert orc.haversine_km(pair[2], pair[3], pair[0], pair[1]) == 0.0


def test_inputs_reach_both_clamps():
    """The placements above are only a test of the clamps if `a` leaves [0, 1] for some of them."""
    a_anti = [restated_a(*p) for p in PLACEMENTS["antipodes"]]
    a_twice = [restated_a(*p) for p in PLACEMENTS["twice_written"]]
    assert sum(a > 1.0 for a in a_anti) >= 1
    assert sum(a < 0.0 for a in a_twice) >= 1
    for p in PLACEMENTS["antipodes"]:
        assert orc.haversine_km(*p) <= HALF_CIRCUMFERENCE_KM    # clamped a = 1 is exactly R·π (rounded)


def test_latitude_pruning_bound_holds():
    """The lemma the latitude-pruned sweeps rest on (pm_proximity_grid.cuh pg_lat_bound, the checker's banded mode):
    for real latitudes, haversine ≥ R·|Δφ|·(1 − 1e-9) − 1e-9.  On the seed's own meridian the two sides are equal in
    exact arithmetic, so half the samples are same-meridian pairs."""
    rng = np.random.default_rng(21)
    n = 60_000
    lat1 = rng.uniform(-90, 90, n)
    lat2 = np.where(rng.random(n) < 0.1, lat1 + rng.normal(0, 1e-3, n), rng.uniform(-90, 90, n)).clip(-90, 90)
    lat1[:4], lat2[:4] = [90.0, -90.0, 0.0, 89.0], [-90.0, 90.0, 90.0, 89.0]
    lon1 = rng.uniform(-180, 180, n)
    same = rng.random(n) < 0.5
    lon2 = np.where(same, lon1, rng.uniform(-180, 180, n))
    worst = -np.inf
    for i in range(n):
        d = orc.haversine_km(lat1[i], lon1[i], lat2[i], lon2[i])
        lb = R * (abs(lat2[i] - lat1[i]) * RADS_PER_DEG)
        assert d >= lb * (1.0 - 1e-9) - 1e-9, (lat1[i], lon1[i], lat2[i], lon2[i], d, lb)
        if same[i]:
            worst = max(worst, lb - d)
    print(f"\n[pruning] largest R·|Δφ| − d on a meridian: {worst:.3e} km")
