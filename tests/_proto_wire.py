"""TEST-ONLY: a Python restatement of the wire-format entry (gub_submit_proto_async): protobuf-go's decoding of GetRateLimitsReq, the
host layer's per-item rules (csrc/host_v1.cpp prepare_call / finish_call, gubernator.go:183-220) and Go's proto.Marshal of
GetRateLimitsResp, plus message generators.  Field numbers are gubernator.proto's: RateLimitReq name 1, unique_key 2, hits 3, limit 4,
duration 5, algorithm 6, behavior 7, burst 8, metadata 9 (map<string, string>), created_at 10 (optional); RateLimitResp status 1,
limit 2, remaining 3, reset_time 4, error 5."""
import numpy as np

import oracle_py as O

OK, TOO_LARGE, MALFORMED = 0, 1, 2
MAX_ITEMS = 1000
MAX_FIELD = (1 << 29) - 1
MAX_TAG = (1 << 31) - 1
GROUP_DEPTH = 100
OUT_FACTOR = 24
IS_OWNER = 0x100


class Malformed(Exception):
    pass


# ---- decoding (protobuf-go) -----------------------------------------------------------------------------------------------------
def _varint(b, p, e):
    v = 0
    for k in range(10):
        if p >= e:
            raise Malformed("truncated varint")
        c = b[p]
        p += 1
        if k == 9:
            if c >= 2:
                raise Malformed("varint overflow")
            return v | (c << 63), p
        v |= (c & 0x7F) << (7 * k)
        if c < 0x80:
            return v, p
    raise Malformed("varint overflow")


def _tag(b, p, e, max_num):
    v, p = _varint(b, p, e)
    if (v >> 3) < 1 or (v >> 3) > max_num:
        raise Malformed("bad field number")
    return v >> 3, v & 7, p


def _bytes(b, p, e):
    n, p = _varint(b, p, e)
    if n > e - p:
        raise Malformed("length past the end")
    return p, p + n


def _skip(b, p, e, num, wt):
    open_ = []
    while True:
        if wt == 0:
            _, p = _varint(b, p, e)
        elif wt in (1, 5):
            w = 8 if wt == 1 else 4
            if e - p < w:
                raise Malformed("truncated fixed")
            p += w
        elif wt == 2:
            _, p = _bytes(b, p, e)
        elif wt == 3:
            if len(open_) == GROUP_DEPTH:
                raise Malformed("groups nested too deep")
            open_.append(num)
        elif wt == 4:
            if not open_ or open_[-1] != num:
                raise Malformed("unmatched end group")
            open_.pop()
        else:
            raise Malformed("bad wire type")
        if not open_:
            return p
        num, wt, p = _tag(b, p, e, MAX_TAG)


def _utf8(raw):
    try:
        raw.decode("utf-8", errors="strict")  # rejects overlong forms, surrogates and > U+10FFFF, as Go's utf8.Valid
    except UnicodeDecodeError:
        raise Malformed("invalid UTF-8")


def _s64(v):
    return v - (1 << 64) if v >= 1 << 63 else v


def _s32(v):
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >= 1 << 31 else v


def decode_item(b, p, e):
    f = dict(name=b"", unique_key=b"", hits=0, limit=0, duration=0, algorithm=0, behavior=0, burst=0, created_at=None)
    while p < e:
        num, wt, p = _tag(b, p, e, MAX_FIELD)
        if num in (1, 2, 9) and wt == 2:
            s, p = _bytes(b, p, e)
            if num == 9:
                q = s
                while q < p:
                    n2, w2, q = _tag(b, q, p, MAX_FIELD)
                    if n2 in (1, 2) and w2 == 2:
                        s2, q = _bytes(b, q, p)
                        _utf8(bytes(b[s2:q]))
                    else:
                        q = _skip(b, q, p, n2, w2)
            else:
                _utf8(bytes(b[s:p]))
                f["name" if num == 1 else "unique_key"] = bytes(b[s:p])
        elif wt == 0 and 3 <= num <= 10 and num != 9:
            v, p = _varint(b, p, e)
            key = {3: "hits", 4: "limit", 5: "duration", 6: "algorithm", 7: "behavior", 8: "burst", 10: "created_at"}[num]
            f[key] = _s32(v) if num in (6, 7) else _s64(v)
        else:
            p = _skip(b, p, e, num, wt)
    return f


def decode_message(msg):
    """(status, [item dicts]) of one GetRateLimitsReq."""
    b = memoryview(msg)
    p, e, items = 0, len(msg), []
    try:
        while p < e:
            num, wt, p = _tag(b, p, e, MAX_FIELD)
            if num == 1 and wt == 2:
                s, p = _bytes(b, p, e)
                items.append(decode_item(b, s, p))
            else:
                p = _skip(b, p, e, num, wt)
    except Malformed:
        return MALFORMED, []
    if len(items) > MAX_ITEMS:
        return TOO_LARGE, []
    return OK, items


# ---- the host layer's rules ---------------------------------------------------------------------------------------------------
def prepare(messages, created):
    """The evaluated batch (O.HREQ_DTYPE) and, per message, (status, [(item, batch index | -code, key)])."""
    rows, plan = [], []
    for msg, dflt in zip(messages, created):
        st, items = decode_message(msg)
        per = []
        for it in items:
            if not it["unique_key"]:
                per.append((it, -1, b""))
            elif not it["name"]:
                per.append((it, -2, b""))
            else:
                key = it["name"] + b"_" + it["unique_key"]
                ca = it["created_at"] if it["created_at"] else dflt
                rows.append((O.xxh64(key), O.fnv1_64(key), it["hits"], it["limit"], it["duration"], it["burst"], ca,
                             it["algorithm"] & 0xFFFFFFFF, (it["behavior"] & 0xFF) | IS_OWNER))
                per.append((it, len(rows) - 1, key))
        plan.append((st, per))
    batch = np.zeros(len(rows), dtype=O.HREQ_DTYPE)
    for i, r in enumerate(rows):
        for name, v in zip(("key_xxh64", "key_fnv1", "hits", "limit", "duration", "burst", "created_at", "algorithm", "behavior"), r):
            batch[i][name] = v
    return batch, plan


def error_text(code, key, algorithm):
    """gub_format_error (csrc/host_v1.cpp), in full."""
    if code == 1:
        return b"field 'unique_key' cannot be empty"
    if code == 2:
        return b"field 'namespace' cannot be empty"
    if code not in (3, 4, 5, 6):
        return b""
    head = b"Error while apply rate limit for '" + key + b"': during workerPool.GetRateLimit: "
    if code == 3:
        return head + b"Invalid rate limit algorithm '%d'" % algorithm
    if code == 6:
        return head + b"rate limit table is full"
    scope = b"Error in leakyBucket" if algorithm == 1 else b"Error in tokenBucket"
    if code == 4:
        return head + scope + b": `Duration = GregorianWeeks` not yet supported; consider making a PR!`"
    return head + scope + b": behavior DURATION_IS_GREGORIAN is set; but `Duration` is not a valid gregorian interval"


# ---- encoding (proto.Marshal) ---------------------------------------------------------------------------------------------------
def varint(v):
    v &= (1 << 64) - 1
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def encode_resp(status=0, limit=0, remaining=0, reset_time=0, error=b""):
    body = b""
    for fnum, v in ((1, status), (2, limit), (3, remaining), (4, reset_time)):
        if v:
            body += bytes([fnum << 3]) + varint(v)
    if error:
        body += b"\x2a" + varint(len(error)) + error
    return b"\x0a" + varint(len(body)) + body


def expected(messages, created, evaluate):
    """[(status, response bytes)] per message; evaluate(batch) -> responses (O.HRESP_DTYPE-like: status, err_code, limit, remaining,
    reset_time) of the batch evaluated in order."""
    batch, plan = prepare(messages, created)
    resp = evaluate(batch) if len(batch) else []
    out = []
    for st, per in plan:
        b = b""
        for it, j, key in per:
            if j < 0:
                b += encode_resp(error=error_text(-j, b"", 0))
                continue
            r = resp[j]
            if int(r["err_code"]):
                b += encode_resp(error=error_text(int(r["err_code"]), key, it["algorithm"]))
            else:
                b += encode_resp(int(r["status"]), int(r["limit"]), int(r["remaining"]), int(r["reset_time"]))
        out.append((st, b))
    return out


# ---- message construction and generators ---------------------------------------------------------------------------------------
def field(num, wt, payload):
    return varint((num << 3) | wt) + payload


def fbytes(num, raw):
    return field(num, 2, varint(len(raw)) + raw)


def fvarint(num, v):
    return field(num, 0, varint(v))


def item(name=b"", unique_key=b"", hits=0, limit=0, duration=0, algorithm=0, behavior=0, burst=0, created_at=None, metadata=(),
         extra=b""):
    """RateLimitReq bytes as a Go client writes them (zero scalars omitted) plus `extra` appended."""
    b = b""
    if name:
        b += fbytes(1, name)
    if unique_key:
        b += fbytes(2, unique_key)
    for num, v in ((3, hits), (4, limit), (5, duration), (6, algorithm), (7, behavior), (8, burst)):
        if v:
            b += fvarint(num, v)
    for k, v in metadata:
        b += fbytes(9, fbytes(1, k) + fbytes(2, v))
    if created_at is not None:
        b += fvarint(10, created_at)
    return b + extra


def message(items, extra=b""):
    return b"".join(fbytes(1, it) for it in items) + extra


def random_items(rng, n, n_keys=1000, zipf=1.1, name=b"proto"):
    ids = np.minimum(rng.zipf(zipf, n), n_keys) - 1
    out = []
    for i in ids.tolist():
        alg = int(rng.integers(0, 2))
        beh = int(rng.choice([0, 0, 0, 8, 32, 4, 1]))
        dur = int(rng.choice([60000, 1000, 3600000])) if beh != 4 else int(rng.integers(0, 6))
        hits = int(rng.choice([1, 1, 1, 0, 2, 5, -1]))
        out.append(item(name, b"k%09d" % i, hits=hits, limit=int(rng.choice([10, 100, 1000])), duration=dur, algorithm=alg,
                        behavior=beh, burst=int(rng.choice([0, 0, 50]))))
    return out


UNPINNED = "unpinned"  # cases where protobuf-go and the Python runtime may disagree (DESIGN.md): never fed to google.protobuf


def edge_messages(rng, now):
    """(name, message bytes, pinned) cases of every rule; pinned=False marks a parity-unpinned case."""
    k = lambda i: item(b"edge", b"e%d" % i, hits=1, limit=5, duration=60000)
    cases = [
        ("empty", b"", True),
        ("zero-length item", message([b""]), True),
        ("empty unique_key", message([item(b"n", b"", hits=1)]), True),
        ("empty name", message([item(b"", b"u", hits=1)]), True),
        ("both empty", message([item()]), True),
        ("repeated scalars", message([item(b"edge", b"r", limit=5, duration=60000, extra=fvarint(3, 1) + fvarint(3, 3) + fvarint(4, 9))]), True),
        ("repeated name", message([fbytes(1, b"first") + fbytes(2, b"u") + fbytes(1, b"second") + fvarint(3, 1) + fvarint(4, 3)
                                   + fvarint(5, 1000)]), True),
        ("unknown varint", message([k(1) + fvarint(99, 7)]), True),
        ("unknown fixed64", message([k(2) + field(20, 1, b"12345678")]), True),
        ("unknown fixed32", message([k(3) + field(21, 5, b"1234")]), True),
        ("unknown bytes", message([k(4) + fbytes(22, b"xyz")]), True),
        ("unknown group", message([k(5) + field(23, 3, fvarint(1, 5) + field(24, 3, b"" ) + field(24, 4, b"")) + field(23, 4, b"")]), True),
        ("top-level unknown", message([k(6)], extra=fvarint(2, 5) + fbytes(3, b"zz")), True),
        ("wrong wire type name", message([k(7) + field(1, 0, varint(5))]), True),
        ("wrong wire type hits", message([k(8) + fbytes(3, b"abc")]), True),
        ("wrong wire type item", message([k(9)], extra=field(1, 0, varint(3))), True),
        ("metadata", message([item(b"edge", b"m", hits=1, limit=5, duration=1000, metadata=[(b"a", b"b"), (b"", b""), (b"k", b"\xc3\xa9")])]), True),
        ("metadata unknown in entry", message([k(10) + fbytes(9, fbytes(1, b"a") + fvarint(3, 1) + field(2, 0, varint(1)))]), True),
        ("metadata wrong wire type", message([k(11) + fvarint(9, 4)]), True),
        ("negative enum", message([item(b"edge", b"ne", hits=1, limit=5, duration=1000, algorithm=-1, behavior=-3)]), True),
        ("big enum", message([item(b"edge", b"be", hits=1, limit=5, duration=1000, algorithm=(1 << 33) + 1)]), True),
        ("invalid algorithm", message([item(b"edge", b"ia", hits=1, limit=5, duration=1000, algorithm=7)]), True),
        ("gregorian weeks", message([item(b"edge", b"gw", hits=1, limit=5, duration=4, behavior=4)]), True),
        ("gregorian invalid", message([item(b"edge", b"gi", hits=1, limit=5, duration=9, behavior=4, algorithm=1)]), True),
        ("created_at zero", message([item(b"edge", b"c0", hits=1, limit=5, duration=1000, created_at=0)]), True),
        ("created_at set", message([item(b"edge", b"c1", hits=1, limit=5, duration=1000, created_at=now - 5000)]), True),
        ("created_at negative", message([item(b"edge", b"c2", hits=1, limit=5, duration=1000, created_at=-7)]), True),
        ("negative hits", message([item(b"edge", b"nh", hits=-5, limit=5, duration=1000)]), True),
        ("10-byte varint", message([item(b"edge", b"v10", hits=1, limit=-1, duration=1000)]), True),
        ("padded varint", message([fbytes(1, b"edge") + fbytes(2, b"pv") + field(3, 0, b"\x81\x80\x80\x00") + fvarint(4, 5) + fvarint(5, 1000)]), True),
        ("key over 255 bytes", message([item(b"edge", b"L" * 400, hits=1, limit=5, duration=1000, algorithm=9)]), True),
        ("name with NUL", message([item(b"ed\x00ge", b"nul", hits=1, limit=5, duration=1000, algorithm=5)]), True),
        ("utf8 name", message([item("naïve".encode(), "ключ".encode(), hits=1, limit=5, duration=1000)]), True),
        # malformed
        ("11-byte varint", message([fbytes(1, b"a") + fbytes(2, b"b") + field(3, 0, b"\xff" * 10 + b"\x01")]), True),
        ("truncated varint", message([fbytes(1, b"a") + field(3, 0, b"\xff\xff")]), True),
        ("length past item", message([fbytes(1, b"a") + field(2, 2, b"\x09ab")]), True),
        ("length past message", field(1, 2, b"\x20" + k(12)), True),
        ("truncated fixed64", message([k(13) + field(20, 1, b"123")]), True),
        ("invalid utf8 name", message([item(b"a\xffb", b"u", hits=1)]), True),
        ("overlong utf8", message([item(b"a", b"\xc0\xaf", hits=1)]), True),
        ("surrogate utf8", message([item(b"a", b"\xed\xa0\x80", hits=1)]), True),
        ("invalid utf8 overwritten", message([fbytes(1, b"\xff") + fbytes(1, b"ok") + fbytes(2, b"u")]), True),
        ("invalid utf8 metadata key", message([k(14) + fbytes(9, fbytes(1, b"\xfe") + fbytes(2, b"v"))]), True),
        ("invalid utf8 metadata value", message([k(15) + fbytes(9, fbytes(1, b"k") + fbytes(2, b"\x80"))]), True),
        ("field number 0", message([k(16) + b"\x00\x01"]), True),
        ("wire type 7", message([k(17) + b"\x0f"]), True),
        ("stray end group", message([k(18) + field(30, 4, b"")]), True),
        ("unclosed group", message([k(19) + field(30, 3, b"")]), True),
        ("mismatched group", message([k(20) + field(30, 3, b"") + field(31, 4, b"")]), True),
        ("malformed item past 1000", message([k(21)] * 1000 + [b"\xff"]), True),
        # the 10th varint byte above 1: protobuf-go rejects it (overflow); upb keeps the low 64 bits
        ("10th varint byte 2", message([fbytes(1, b"a") + fbytes(2, b"b") + field(3, 0, b"\xff" * 9 + b"\x02")]), False),
        # field numbers above 2^29 - 1 inside a group: protobuf-go's ConsumeTag takes them
        ("group field number 2^30", message([k(22) + field(30, 3, varint(((1 << 30) << 3) | 0) + b"\x01") + field(30, 4, b"")]), False),
    ]
    deep = field(40, 3, b"") * 101 + field(40, 4, b"") * 101
    cases.append(("groups nested 101 deep", message([k(23) + deep]), False))
    return cases


def sized_messages(rng):
    """Exactly 1000 items, 1001 items, and the output bound's worst cases."""
    it = item(b"sz", b"s", hits=1, limit=3, duration=1000)
    return [
        ("1000 items", message([it] * 1000)),
        ("1001 items", message([it] * 1001)),
        ("1000 empty items", message([b""] * 1000)),
        ("1000 gregorian errors", message([item(b"a", b"b", duration=9, behavior=4)] * 1000)),
        # (the oracle's hashed entry keeps the algorithm's low byte only: an invalid algorithm must be invalid there too)
        ("1000 invalid algorithms", message([item(b"a", b"b", algorithm=-2147483646)] * 1000)),
    ]
