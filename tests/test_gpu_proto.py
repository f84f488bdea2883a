"""gub_submit_proto_async on the H100: GetRateLimitsReq wire bytes in, GetRateLimitsResp wire bytes out, checked byte for byte against the
restatement's encoding (tests/_proto_wire.py) of what the host layer (gub_instance_get_rate_limits_unbounded on a twin table) returns for
the same items, with both tables' scans and counters compared."""
import numpy as np
import pytest

import _proto_wire as W
from workloads import T0

pytestmark = pytest.mark.gpu

GUARD = 256
N_KEYS = 1 << 20


@pytest.fixture(scope="module")
def G():
    import gubernator_b200 as g
    return g


class Call:
    """One call's page-locked buffers, with GUARD bytes of 0xA5 before and after each output."""

    def __init__(self, G, messages, now):
        self.G, self.messages, self.n = G, messages, len(messages)
        packed, self.bound = G.native.pack_proto(messages, now)
        self.pk = G.native.PinnedArray(len(packed), np.uint8)
        self.pk.array[:] = packed
        self.out = G.native.PinnedArray(self.bound + 2 * GUARD, np.uint8)
        self.off = G.native.PinnedArray(self.n + 1 + 2 * GUARD // 8, np.uint64)
        self.st = G.native.PinnedArray(self.n + 2 * GUARD // 4, np.uint32)
        for a in (self.out, self.off, self.st):
            a.array.view(np.uint8)[:] = 0xA5

    def submit(self, tab, clk):
        a = lambda p, k: p.ptr + k
        return tab.submit_proto_async(self.pk.ptr, len(self.pk.array), self.n, clk, a(self.out, GUARD), self.bound,
                                      a(self.off, GUARD), a(self.st, GUARD))

    def result(self):
        for a in (self.out, self.off, self.st):
            b = a.array.view(np.uint8)
            assert (b[:GUARD] == 0xA5).all() and (b[len(b) - GUARD:] == 0xA5).all(), "a guard byte was overwritten"
        off = self.off.array[GUARD // 8:GUARD // 8 + self.n + 1]
        out = self.out.array[GUARD:GUARD + self.bound]
        return self.st.array[GUARD // 4:GUARD // 4 + self.n].tolist(), [out[int(off[m]):int(off[m + 1])].tobytes() for m in range(self.n)]

    def free(self):
        for a in (self.pk, self.out, self.off, self.st):
            a.free()


def host_layer(inst, messages, now):
    """What the host layer answers for the call's OK messages as one unbounded call (the aggregator's batch), encoded per message."""
    plan = [W.decode_message(m) for m in messages]
    reqs = [dict(name=it["name"].decode(), unique_key=it["unique_key"].decode(), hits=it["hits"], limit=it["limit"],
                 duration=it["duration"], burst=it["burst"], algorithm=it["algorithm"], behavior=it["behavior"],
                 created_at=it["created_at"] or 0) for st, items in plan for it in items]
    inst.set_now(now)
    resp = inst.get_rate_limits(reqs, unbounded=True) if reqs else []
    out, k = [], 0
    for st, items in plan:
        b = b""
        for _ in items:
            r = resp[k]
            k += 1
            b += W.encode_resp(r["status"], r["limit"], r["remaining"], r["reset_time"], r["error"].encode())
        out.append((st, b))
    return out


def traffic(rng, n_msgs=100, items=65536, bad=True):
    sizes = rng.multinomial(items, np.full(n_msgs, 1.0 / n_msgs))
    msgs = [W.message(W.random_items(rng, int(min(s, 1000)), n_keys=N_KEYS)) for s in sizes]
    if bad:
        msgs[7] = W.message([W.item(b"x", b"y", hits=1)] * 1001)
        msgs[n_msgs // 2] = W.message([W.item(b"x", b"\xff")])
        msgs[-1] = W.message([W.item(b"", b"u", hits=1), W.item(b"n", b"", hits=1), b""])
    return msgs


def _scan(tab):
    s = tab.scan()
    return np.sort(s, order=["key_xxh64", "key_fnv1"])


def _same_tables(a, b):
    sa, sb = _scan(a), _scan(b)
    assert len(sa) == len(sb) and sa.tobytes() == sb.tobytes()
    assert a.counters() == b.counters()


def test_calls_match_host_layer_on_a_twin_table(G):
    from gubernator_b200.service import V1Instance
    rng = np.random.default_rng(11)
    tab = G.Table(1 << 22)
    twin = V1Instance(table=G.Table(1 << 22))
    for c in range(4):
        now = T0 + 900 * c
        msgs = traffic(rng)
        call = Call(G, msgs, now)
        tab.wait(call.submit(tab, G.clock_fill(now)))
        st, outs = call.result()
        want = host_layer(twin, msgs, now)
        assert st == [s for s, _ in want]
        assert st[7] == W.TOO_LARGE and st[50] == W.MALFORMED
        for m, (b, (_, wb)) in enumerate(zip(outs, want)):
            assert b == wb, f"call {c} message {m}: response bytes differ"
        call.free()
    _same_tables(tab, twin.table)


def test_pipelined_calls_equal_calls_one_by_one(G):
    rng = np.random.default_rng(12)
    a, b = G.Table(1 << 21), G.Table(1 << 21)
    depth = G.native.lib().gub_pipeline_depth(a._h)
    calls = [(T0 + 500 * c, traffic(rng, n_msgs=40, items=20000)) for c in range(2 * depth)]
    one = []
    for now, msgs in calls:
        call = Call(G, msgs, now)
        a.wait(call.submit(a, G.clock_fill(now)))
        one.append(call.result())
        call.free()
    piped, inflight = [], []
    for now, msgs in calls:
        if len(inflight) == depth:
            call, tk = inflight.pop(0)
            b.wait(tk)
            piped.append(call.result())
            call.free()
        call = Call(G, msgs, now)
        inflight.append((call, call.submit(b, G.clock_fill(now))))
    for call, tk in inflight:
        b.wait(tk)
        piped.append(call.result())
        call.free()
    assert piped == one
    _same_tables(a, b)


def test_rejected_messages_leave_the_table_unchanged(G):
    rng = np.random.default_rng(13)
    tab = G.Table(1 << 16)
    warm = Call(G, traffic(rng, n_msgs=10, items=3000, bad=False), T0)
    tab.wait(warm.submit(tab, G.clock_fill(T0)))
    warm.free()
    before, counters = _scan(tab), tab.counters()
    bad = [W.message([W.item(b"x", b"y", hits=1)] * 1001)] + [m for n, m, _ in W.edge_messages(rng, T0)
                                                               if W.decode_message(m)[0] == W.MALFORMED]
    call = Call(G, bad, T0 + 10)
    tab.wait(call.submit(tab, G.clock_fill(T0 + 10)))
    st, outs = call.result()
    assert st[0] == W.TOO_LARGE and all(s == W.MALFORMED for s in st[1:]) and all(o == b"" for o in outs)
    call.free()
    assert _scan(tab).tobytes() == before.tobytes()
    after = tab.counters()
    assert after == counters


def test_plain_host_memory_is_refused(G):
    tab = G.Table(1 << 12)
    packed, bound = G.native.pack_proto([W.message([W.item(b"a", b"b", hits=1)])], T0)
    out, off, st = np.zeros(bound, np.uint8), np.zeros(2, np.uint64), np.zeros(1, np.uint32)
    with pytest.raises(G.native.GubError, match="page-locked"):
        tab.submit_proto_async(packed.ctypes.data, len(packed), 1, G.clock_fill(T0), out.ctypes.data, bound, off.ctypes.data, st.ctypes.data)
