"""The device build of bucket_math.cuh (tests/bucket_math_dev.cu, the product library's nvcc flags) against its host build
(tests/host_math_harness.cpp, itself pinned to the oracle by test_host_math.py), bit for bit: f2i() on every edge double and a
million random bit patterns, apply_one() and run_to_rank() on a million lattice (state, request) pairs from edge_states.py.

The host build compiles f2i()'s CVTTSD2SI branch and SSE2 arithmetic; only these tests and the GPU pipeline run the device branch
and the device's float64 unit.  A mismatch message carries what add.f64 returned for NaN operands on this device."""
import numpy as np
import pytest

import edge_states as ES
import oracle_py as O
import _host_math as H
from workloads import make_clock

pytestmark = pytest.mark.gpu


def _edge_doubles(rng):
    xs = []
    for m in (2.0 ** 52, 2.0 ** 53, 2.0 ** 63):
        for v in (m, -m):
            xs += [v, np.nextafter(v, np.inf), np.nextafter(v, -np.inf)]
    xs += [0.0, -0.0, 5e-324, -5e-324, 2.2250738585072009e-308, -2.2250738585072009e-308, np.inf, -np.inf, 0.5, -0.5, 1.0, -1.0]
    bits = [ES.fbits(x) for x in xs] + ES.LEAKY_REMAINING
    for sign in (0, 1 << 63):
        for quiet in (0, 1 << 51):
            for payload in (1, 2, 0xDEADBEEF, (1 << 50) - 1, 1 << 50):
                if quiet or payload:
                    bits.append(sign | 0x7FF0000000000000 | quiet | payload)
            if quiet:
                bits.append(sign | 0x7FF0000000000000 | quiet)
    bits = np.concatenate([np.array(bits, dtype=np.uint64), rng.integers(0, 1 << 64, 1 << 20, dtype=np.uint64)])
    return bits.view(np.float64)


def _nan_add_probe():
    """What add.f64 returns on this device for NaN operands, next to SSE2's answer (numpy on the host CPU)."""
    a = np.array([0x7FF80000DEADBEEF, 0x7FF0000000000001, ES.fbits(1.0), 0xFFF80000DEADBEEF, ES.fbits(-np.inf)], dtype=np.uint64)
    b = np.array([ES.fbits(1.0), ES.fbits(5.0), 0x7FF800000000ABCD, 0x7FF800000000ABCD, ES.fbits(np.inf)], dtype=np.uint64)
    dev = np.zeros(len(a), dtype=np.uint64)
    L = H.dev_lib()
    L.bmd_add(a.ctypes.data, b.ctypes.data, dev.ctypes.data, len(a))
    with np.errstate(invalid="ignore"):
        host = (a.view(np.float64) + b.view(np.float64)).view(np.uint64)
    return "; ".join(f"{x:#018x} + {y:#018x}: device {d:#018x}, SSE2 {h:#018x}" for x, y, d, h in zip(a, b, dev, host))


def _first_mismatch(what, dev, host, inputs):
    bad = np.nonzero(dev != host)[0]
    if len(bad) == 0:
        return
    i = int(bad[0])
    fields = [f for f in (dev.dtype.names or ()) if dev[f][i] != host[f][i]] if dev.dtype.names else [""]
    raise AssertionError(f"{what}: {len(bad)} of {len(dev)} differ; first at {i}, fields {fields}: device {dev[i]} host {host[i]}; "
                         f"inputs {[x[i] for x in inputs]}; add.f64 on NaN: {_nan_add_probe()}")


def _rem_view(b):
    """Slot images with the float64 Remaining kept as bits (BUCKET_DTYPE already stores it as uint64) and no padding."""
    return b[[f for f in b.dtype.names if f != "_pad"]]


def test_f2i_device_equals_host():
    x = _edge_doubles(np.random.default_rng(1))
    dev, host = H.f2i(H.dev_lib(), x), H.f2i(H.lib(), x)
    _first_mismatch("f2i", dev, host, [x.view(np.uint64)])


def test_f2i_control_bare_conversion_disagrees():
    """The lattice is strong enough to see the patch: the saturating cvt.rzi alone must disagree with CVTTSD2SI on it."""
    x = _edge_doubles(np.random.default_rng(2))
    bare, host = H.f2i(H.dev_lib(), x, "bmd_f2i_bare"), H.f2i(H.lib(), x)
    bad = bare != host
    assert bad.any()
    assert np.all(np.isnan(x[bad]) | (x[bad] >= 2.0 ** 63)), "the bare conversion differs only where f2i patches it"


@pytest.mark.parametrize("seed", range(2))
def test_apply_one_device_equals_host(seed):
    rng = np.random.default_rng(300 + seed)
    b, rq, _, _ = ES.pairs(rng, 1 << 19, H.BUCKET_DTYPE, O.HREQ_DTYPE)
    clk = make_clock(ES.NOW)
    dr, db, dd = H.apply_one(H.dev_lib(), b, rq, clk)
    hr, hb, hd = H.apply_one(H.lib(), b, rq, clk)
    _first_mismatch("apply_one response", dr, hr, [b, rq])
    _first_mismatch("apply_one state", _rem_view(db), _rem_view(hb), [b, rq])
    _first_mismatch("apply_one counters", dd, hd, [b, rq])


@pytest.mark.parametrize("seed", range(2))
def test_run_to_rank_device_equals_host(seed):
    rng = np.random.default_rng(400 + seed)
    b, rq, t, _ = ES.pairs(rng, 1 << 19, H.BUCKET_DTYPE, O.HREQ_DTYPE)
    clk = make_clock(ES.NOW)
    dr, db, dd = H.run_to_rank(H.dev_lib(), b, rq, t, clk)
    hr, hb, hd = H.run_to_rank(H.lib(), b, rq, t, clk)
    _first_mismatch("run_to_rank response", dr, hr, [b, rq, t])
    _first_mismatch("run_to_rank state", _rem_view(db), _rem_view(hb), [b, rq, t])
    _first_mismatch("run_to_rank counters", dd, hd, [b, rq, t])
