"""CPU: the weighted EBU R128 restatement (tests/_ebu_weighted.cc, the oracle of the weighted EBUr128 banks) and the BS.1770-4
position rule.

 * the restatement with the reference's own weights (mono {2}, else 1 1 1 1.41 1.41) must be Ebu_r128_proc itself, bit for
   bit, so that the weighted GPU tests compare against a restatement that is exact where the reference exists;
 * b200m_bs1770_weights (host only: no device needed) gives 1.41 for |elevation| < 30 and 60 <= |azimuth| <= 120, else 1.0.
"""
import numpy as np
import pytest

import _ebu_weighted as W
import _oracle as O

DEFAULT = {1: [2.0], 2: [1, 1], 3: [1, 1, 1], 4: [1, 1, 1, 1.41], 5: [1, 1, 1, 1.41, 1.41]}


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _block(rng, rows, n):
    """noise at per-row levels, with NaN, +-Inf, denormals and exact zeros sprinkled in"""
    x = (rng.standard_normal((rows, n)) * 10.0 ** rng.uniform(-4, 0, (rows, 1))).astype(np.float32)
    if n > 8:
        for _ in range(3):
            r, j = int(rng.integers(rows)), int(rng.integers(n))
            x[r, j] = rng.choice([np.nan, np.inf, -np.inf])
        r = int(rng.integers(rows))
        x[r, : n // 2] = np.float32(1e-41) * rng.choice([-1, 1], n // 2)      # subnormal input
        x[int(rng.integers(rows))] = 0.0
    return x


@pytest.mark.skipif(not O.available("reference"), reason="needs the reference oracle (oracle/_ref)")
@pytest.mark.parametrize("nchan", [1, 2, 3, 4, 5])
def test_weighted_restatement_is_the_reference_with_default_gains(nchan):
    n_inst = 7
    rng = np.random.default_rng(40 + nchan)
    ref = O.Ebu(n_inst, nchan, kind="reference")
    w = W.Ebu(n_inst, DEFAULT[nchan])
    for e in (ref, w):
        e.integr("start")
    for b in range(120):
        if b % 17 == 5:
            i = int(rng.integers(n_inst))
            cmd = ("pause", "start", "reset", "new")[int(rng.integers(4))]
            for e in (ref, w):
                if cmd == "new":
                    e.reset(i)
                else:
                    e.integr(cmd, i)
        n = int(rng.choice([1, 7, 64, 480, 1000, 1024, 2400, 4097, 8192]))
        x = _block(rng, n_inst * nchan, n)
        ref.process(x); w.process(x)
        assert np.array_equal(u32(ref.read()), u32(w.read())), (nchan, b)
    for i in range(n_inst):
        a, b = ref.hist(i), w.hist(i)
        for p, q in zip(a, b):
            assert np.array_equal(p, q), (nchan, i)


def _weights(az, el):
    import meters_lv2_b200 as B
    return B.bs1770_weights(az, el)


def test_bs1770_weights_5_0():
    g = _weights([-30, 30, 0, -110, 110], [0, 0, 0, 0, 0])
    assert g.tolist() == np.float32([1, 1, 1, 1.41, 1.41]).tolist()


def test_bs1770_weights_7_1_4():
    # L R C (LFE left out) Lss Rss Lrs Rrs, then four heights at 30..45 degrees elevation
    az = [30, -30, 0, 90, -90, 135, -135, 45, -45, 135, -135]
    el = [0, 0, 0, 0, 0, 0, 0, 30, 35, 45, 40]
    g = _weights(az, el)
    want = np.ones(11, np.float32); want[3:5] = 1.41
    assert g.tolist() == want.tolist()


def test_bs1770_weights_edges_and_signs():
    g = _weights([60, 120, -60, -120, 59.9, 120.1, 90, 90, 90, 250, -290], [0, 0, 0, 0, 0, 0, 30, -30, -29.9, 0, 0])
    assert g.tolist() == np.float32([1.41, 1.41, 1.41, 1.41, 1, 1, 1, 1, 1.41, 1.41, 1.41]).tolist()


def test_bs1770_weights_rejects_non_finite():
    import meters_lv2_b200 as B
    with pytest.raises(B.B200MError):
        _weights([0, np.nan], [0, 0])
    with pytest.raises(B.B200MError):
        _weights([0, 0], [np.inf, 0])
