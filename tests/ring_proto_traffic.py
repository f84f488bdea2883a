"""TEST-ONLY: RPC traffic for the tests of GetRateLimits wire bytes on the ring.  _proto_wire.random_items' mix of items, with unique
keys whose FNV-1 spreads them over the ring's shards: keys that differ only in their last few bytes share the top bits of FNV-1, so a
few hundred keys of the form "k%09d" all land on one or two owners."""
import numpy as np

import _proto_wire as W

PEER_TIMEOUT = 7  # GUB_ERR_PEER_TIMEOUT


def spread_items(rng, n, n_keys=1000, zipf=1.1, name=b"ring"):
    ids = np.minimum(rng.zipf(zipf, n), n_keys) - 1
    out = []
    for i in ids.tolist():
        alg = int(rng.integers(0, 2))
        beh = int(rng.choice([0, 0, 0, 8, 32, 4, 1]))
        dur = int(rng.choice([60000, 1000, 3600000])) if beh != 4 else int(rng.integers(0, 6))
        hits = int(rng.choice([1, 1, 1, 0, 2, 5, -1]))
        out.append(W.item(name, (b"%09d" % i)[::-1] + b"k", hits=hits, limit=int(rng.choice([10, 100, 1000])), duration=dur, algorithm=alg,
                          behavior=beh, burst=int(rng.choice([0, 0, 50]))))
    return out


def error_text(code, key, algorithm):
    """The restatement's gub_format_error plus the ring's code 7 (gubernator.go:374 around a timed-out peer call)."""
    if code == PEER_TIMEOUT:
        return b"Error while fetching rate limit '" + key + b"' from peer: context deadline exceeded"
    return W.error_text(code, key, algorithm)


def encode(plan, resp):
    """[(status, response bytes)] per message of one shard, from its plan (W.prepare) and its dense batch's responses."""
    out = []
    for st, per in plan:
        b = b""
        for it, j, key in per:
            if j < 0:
                b += W.encode_resp(error=W.error_text(-j, b"", 0))
            elif int(resp[j]["err_code"]):
                b += W.encode_resp(error=error_text(int(resp[j]["err_code"]), key, it["algorithm"]))
            else:
                r = resp[j]
                b += W.encode_resp(int(r["status"]), int(r["limit"]), int(r["remaining"]), int(r["reset_time"]))
        out.append((st, b))
    return out
