"""CPU: the wire-format entry's kernels (gub_proto.cuh, emulated through tests/cuda_emu.h) against the Python restatement of its rules
(tests/_proto_wire.py) with the oracle evaluating the batch, and the restatement against google.protobuf where that imports."""
import numpy as np
import pytest

import oracle_py as O
import _proto_wire as W
from _proto_emu import ProtoEmuTable
from workloads import T0, make_clock

import gubernator_b200.native as N

GUARD = 64


def _run(tab, pool, messages, created, now):
    packed, bound = N.pack_proto(messages, created)
    clk = make_clock(now)
    st, outs, raw, _ = tab.submit_proto(packed, len(messages), clk, bound, guard=GUARD)
    pool.set_now(now)
    want = W.expected(messages, created, pool.submit_hashed)
    assert bytes(raw[:GUARD]) == b"\xa5" * GUARD and bytes(raw[GUARD + bound:]) == b"\xa5" * GUARD, "a guard byte was overwritten"
    return st, outs, want, bound


def _check(st, outs, want, names):
    for m, ((ws, wb), s, b) in enumerate(zip(want, st, outs)):
        assert s == ws, f"{names[m]}: status {s}, want {ws}"
        assert b == wb, f"{names[m]}: response bytes differ"


def test_edge_cases_match_restatement_and_oracle():
    tab = ProtoEmuTable(1 << 14, max_batch=4096)
    pool = O.Pool(workers=1, cache_size=1_000_000, now_ms=T0)
    cases = W.edge_messages(np.random.default_rng(1), T0)
    names = [c[0] for c in cases]
    msgs = [c[1] for c in cases]
    created = np.array([T0 - 3 * i for i in range(len(msgs))], dtype=np.int64)
    st, outs, want, _ = _run(tab, pool, msgs, created, T0)
    _check(st, outs, want, names)
    by = dict(zip(names, st))
    for n in ("11-byte varint", "truncated varint", "length past item", "length past message", "invalid utf8 name", "overlong utf8",
              "surrogate utf8", "invalid utf8 overwritten", "invalid utf8 metadata key", "invalid utf8 metadata value", "field number 0",
              "wire type 7", "stray end group", "unclosed group", "mismatched group", "malformed item past 1000", "10th varint byte 2",
              "groups nested 101 deep", "wrong wire type item"):
        assert by[n] == (W.OK if n == "wrong wire type item" else W.MALFORMED), n
    assert by["unknown group"] == W.OK and by["metadata"] == W.OK and by["group field number 2^30"] == W.OK
    # a long key's error text is not cut at 255 bytes
    long = outs[names.index("key over 255 bytes")]
    assert b"L" * 400 in long and len(long) > 400


def test_sizes_and_output_bound():
    tab = ProtoEmuTable(1 << 14, max_batch=1024)
    pool = O.Pool(workers=1, cache_size=1_000_000, now_ms=T0)
    cases = W.sized_messages(np.random.default_rng(2))
    names, msgs = [c[0] for c in cases], [c[1] for c in cases]
    st, outs, want, bound = _run(tab, pool, msgs, np.full(len(msgs), T0, dtype=np.int64), T0)
    _check(st, outs, want, names)
    assert st == [W.OK, W.TOO_LARGE, W.OK, W.OK, W.OK]
    for m, b in zip(msgs, outs):
        assert len(b) <= W.OUT_FACTOR * len(m)
    assert sum(len(b) for b in outs) <= bound


def test_random_traffic_several_calls():
    rng = np.random.default_rng(3)
    tab = ProtoEmuTable(1 << 15, max_batch=1024)
    pool = O.Pool(workers=1, cache_size=1_000_000, now_ms=T0)
    evaluated = 0
    for call in range(3):
        now = T0 + 700 * call
        msgs = []
        for _ in range(12):
            items = W.random_items(rng, int(rng.integers(0, 120)), n_keys=300)
            if rng.random() < 0.2:
                items.insert(int(rng.integers(0, len(items) + 1)), W.item(b"", b"x"))
            msgs.append(W.message(items))
        msgs.insert(4, W.message([W.item(b"bad", b"\xff")]))
        created = np.array([now - int(rng.integers(0, 50)) for _ in msgs], dtype=np.int64)
        st, outs, want, _ = _run(tab, pool, msgs, created, now)
        _check(st, outs, want, [f"call {call} msg {m}" for m in range(len(msgs))])
        evaluated += len(W.prepare(msgs, created)[0])
    assert tab.counters()["requests"] == evaluated


def test_host_checks_refuse_bad_offsets_and_small_out():
    tab = ProtoEmuTable(1 << 10, max_batch=1024)
    msgs = [W.message([W.item(b"a", b"b", hits=1)])]
    packed, bound = N.pack_proto(msgs, T0)
    clk = make_clock(T0)
    with pytest.raises(AssertionError):
        tab.submit_proto(packed, 1, clk, bound - 1)
    bad = packed.copy()
    o_at = 8
    bad[o_at + 4:o_at + 8] = np.frombuffer(np.uint32(len(packed)).tobytes(), dtype=np.uint8)
    with pytest.raises(AssertionError):
        tab.submit_proto(bad, 1, clk, bound)


# ---- google.protobuf: the restatement's rules against a real protobuf runtime ----------------------------------------------------
def _classes():
    pb = pytest.importorskip("google.protobuf")
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    F = descriptor_pb2.FieldDescriptorProto
    fd = descriptor_pb2.FileDescriptorProto(name="proto_wire_test.proto", package="wiretest", syntax="proto3")
    for name, values in (("Algorithm", [("TOKEN_BUCKET", 0), ("LEAKY_BUCKET", 1)]), ("Status", [("UNDER_LIMIT", 0), ("OVER_LIMIT", 1)]),
                         ("Behavior", [("BATCHING", 0), ("NO_BATCHING", 1)])):
        e = fd.enum_type.add(name=name)
        for n, v in values:
            e.value.add(name=n, number=v)
    req = fd.message_type.add(name="RateLimitReq")
    entry = req.nested_type.add(name="MetadataEntry")
    entry.options.map_entry = True
    entry.field.add(name="key", number=1, type=F.TYPE_STRING, label=F.LABEL_OPTIONAL)
    entry.field.add(name="value", number=2, type=F.TYPE_STRING, label=F.LABEL_OPTIONAL)
    for name, num, typ, tn in (("name", 1, F.TYPE_STRING, None), ("unique_key", 2, F.TYPE_STRING, None), ("hits", 3, F.TYPE_INT64, None),
                               ("limit", 4, F.TYPE_INT64, None), ("duration", 5, F.TYPE_INT64, None),
                               ("algorithm", 6, F.TYPE_ENUM, ".wiretest.Algorithm"), ("behavior", 7, F.TYPE_ENUM, ".wiretest.Behavior"),
                               ("burst", 8, F.TYPE_INT64, None)):
        f = req.field.add(name=name, number=num, type=typ, label=F.LABEL_OPTIONAL)
        if tn:
            f.type_name = tn
    req.field.add(name="metadata", number=9, type=F.TYPE_MESSAGE, label=F.LABEL_REPEATED, type_name=".wiretest.RateLimitReq.MetadataEntry")
    req.oneof_decl.add(name="_created_at")
    req.field.add(name="created_at", number=10, type=F.TYPE_INT64, label=F.LABEL_OPTIONAL, oneof_index=0, proto3_optional=True)
    top = fd.message_type.add(name="GetRateLimitsReq")
    top.field.add(name="requests", number=1, type=F.TYPE_MESSAGE, label=F.LABEL_REPEATED, type_name=".wiretest.RateLimitReq")
    resp = fd.message_type.add(name="RateLimitResp")
    resp.field.add(name="status", number=1, type=F.TYPE_ENUM, label=F.LABEL_OPTIONAL, type_name=".wiretest.Status")
    for name, num in (("limit", 2), ("remaining", 3), ("reset_time", 4)):
        resp.field.add(name=name, number=num, type=F.TYPE_INT64, label=F.LABEL_OPTIONAL)
    resp.field.add(name="error", number=5, type=F.TYPE_STRING, label=F.LABEL_OPTIONAL)
    rtop = fd.message_type.add(name="GetRateLimitsResp")
    rtop.field.add(name="responses", number=1, type=F.TYPE_MESSAGE, label=F.LABEL_REPEATED, type_name=".wiretest.RateLimitResp")
    dp = descriptor_pool.DescriptorPool()
    dp.Add(fd)
    get = lambda n: message_factory.GetMessageClass(dp.FindMessageTypeByName("wiretest." + n))
    return get("GetRateLimitsReq"), get("GetRateLimitsResp"), get("RateLimitResp")


def _all_pinned_messages():
    rng = np.random.default_rng(4)
    out = [(n, m) for n, m, pinned in W.edge_messages(rng, T0) if pinned]
    out += W.sized_messages(rng)
    out += [(f"random {k}", W.message(W.random_items(rng, 40))) for k in range(5)]
    return out


def test_restatement_agrees_with_google_protobuf_decoding():
    Req, _, _ = _classes()
    from google.protobuf.message import DecodeError
    for name, msg in _all_pinned_messages():
        st, items = W.decode_message(msg)
        m = Req()
        try:
            m.ParseFromString(msg)
            accepted = True
        except DecodeError:
            accepted = False
        assert accepted == (st != W.MALFORMED), name
        if not accepted:
            continue
        assert len(m.requests) == (len(items) if st == W.OK else len(m.requests)), name
        if st == W.TOO_LARGE:
            assert len(m.requests) > W.MAX_ITEMS, name
            continue
        for r, it in zip(m.requests, items):
            assert r.name.encode() == it["name"] and r.unique_key.encode() == it["unique_key"], name
            for f in ("hits", "limit", "duration", "burst", "algorithm", "behavior"):
                assert getattr(r, f) == it[f], (name, f)
            assert r.HasField("created_at") == (it["created_at"] is not None), name
            if it["created_at"] is not None:
                assert r.created_at == it["created_at"], name


def test_restatement_encoding_equals_serialize_to_string():
    _, Resp, One = _classes()
    pool = O.Pool(workers=1, cache_size=1_000_000, now_ms=T0)
    msgs = [m for _, m in _all_pinned_messages()]
    created = np.full(len(msgs), T0, dtype=np.int64)
    batch, plan = W.prepare(msgs, created)
    resp = pool.submit_hashed(batch)
    want = W.expected(msgs, created, lambda b: resp)
    for (st, per), (_, ours) in zip(plan, want):
        out = Resp()
        for it, j, key in per:
            r = out.responses.add()
            if j < 0:
                r.error = W.error_text(-j, b"", 0).decode()
            elif int(resp[j]["err_code"]):
                r.error = W.error_text(int(resp[j]["err_code"]), key, it["algorithm"]).decode("utf-8", "surrogateescape")
            else:
                r.status, r.limit, r.remaining, r.reset_time = (int(resp[j][f]) for f in ("status", "limit", "remaining", "reset_time"))
        assert out.SerializeToString(deterministic=True) == ours
