"""The flow query tables of GYSK_FLAG_FLOW_QUERIES restated on the CPU (tests only). A response sample counts iff it reaches its service's
response histogram: a GYSK_EV_RESP event of a service that has a slot, value within the RESP validity rule. It adds {1 | msec << 32},
msec = usec / 1000, to the cell of its flow key in every row, at the connection count-min's columns (h1 + r * (h2 | 1)) & wmask with the
two lookup2 words of the key. The hashes are restated here with numpy so that millions of keys cost no call per key; the CPU tests pin
them to the oracle's gyo_cms_index. The raw routes' keys are restated from the decoders: see route_key_*."""
import numpy as np

from gyeeta_b200 import engine as ge

U32 = 0xFFFFFFFF
VALID_USEC = 1000001000          # GYSK_EV_RESP validity rule: response msec <= 1 000 000
GOLDEN, GY_SEED = 0x9E3779B9, 0xCEEDFEAD
SEED_A, SEED_B = GY_SEED, GY_SEED ^ 0x5BD1E995


def jhash_2words(a, b, c):
    """lookup2's jhash_2words on uint32 arrays (gysk_device.cuh)"""
    a = np.asarray(a, dtype=np.uint32) + np.uint32(GOLDEN)
    b = np.asarray(b, dtype=np.uint32) + np.uint32(GOLDEN)
    c = np.broadcast_to(np.asarray(c, dtype=np.uint32), a.shape).copy()
    with np.errstate(over="ignore"):
        for sa, sb, sc in ((13, 8, 13), (12, 16, 5), (3, 10, 15)):
            a = (a - b - c) ^ (c >> np.uint32(sa))
            b = (b - c - a) ^ (a << np.uint32(sb))
            c = (c - a - b) ^ (b >> np.uint32(sc))
    return c


def flow_hashes(keys):
    keys = np.asarray(keys, dtype=np.uint64)
    lo, hi = (keys & np.uint64(U32)).astype(np.uint32), (keys >> np.uint64(32)).astype(np.uint32)
    return jhash_2words(lo, hi, SEED_A), jhash_2words(lo, hi, SEED_B)


def columns(keys, depth, log2w):
    """[depth, n] column of each key in each row"""
    h1, h2 = flow_hashes(keys)
    with np.errstate(over="ignore"):
        return np.stack([(h1 + np.uint32(r) * (h2 | np.uint32(1))) & np.uint32((1 << log2w) - 1) for r in range(depth)]).astype(np.int64)


def counted(ev, known):
    """the samples that reach a histogram: RESP events within the validity rule whose service has a slot (known: set of ids)"""
    m = (ev["type"] == ge.EV_RESP) & (ev["value"] < VALID_USEC)
    ids = ev["svc_id"]
    if known is not None:
        u, inv = np.unique(ids, return_inverse=True)
        m &= np.isin(u, np.fromiter(known, dtype=np.uint64, count=len(known)))[inv.reshape(-1)]
    return ev[m]


def increments(samples):
    return np.uint64(1) | ((samples["value"] // np.uint32(1000)).astype(np.uint64) << np.uint64(32))


def add_samples(table, samples, depth, log2w):
    """table ([depth << log2w] uint64) += the samples' increments, mod 2^64 per cell like RED.ADD.64"""
    if not len(samples):
        return table
    t = table.reshape(depth, 1 << log2w)
    cols, inc = columns(samples["flow_key"], depth, log2w), increments(samples)
    for r in range(depth):
        np.add.at(t[r], cols[r], inc)
    return table


def point_query(table, keys, depth, log2w):
    """gysk_query_flow_queries restated: per key the minimum over rows of each half"""
    t = table.reshape(depth, 1 << log2w)
    cells = np.stack([t[r][c] for r, c in enumerate(columns(keys, depth, log2w))])
    return (cells & np.uint64(U32)).min(axis=0).astype(np.uint32), (cells >> np.uint64(32)).min(axis=0).astype(np.uint32)


def exact(samples, keys):
    """the exact (queries, response msec) of each key, as Python ints"""
    keys = np.asarray(keys, dtype=np.uint64)
    ms = (samples["value"] // np.uint32(1000)).astype(np.uint64)
    u, inv = np.unique(samples["flow_key"], return_inverse=True)
    q = np.bincount(inv.reshape(-1), minlength=len(u))
    s = np.bincount(inv.reshape(-1), weights=ms.astype(np.float64), minlength=len(u))
    pos = np.searchsorted(u, keys)
    hit = (pos < len(u)) & (u[np.minimum(pos, len(u) - 1)] == keys)
    return [(int(q[p]), int(s[p])) if h else (0, 0) for p, h in zip(pos.tolist(), hit.tolist())]


def row_sums(table, depth, log2w):
    """per row the sum of the low (query) halves, mod 2^32"""
    t = table.reshape(depth, 1 << log2w)
    return [int((t[r] & np.uint64(U32)).sum(dtype=np.uint64)) & U32 for r in range(depth)]


# the flow key each raw route gives a response sample (gysk_engine.cu decode_resp / decode_raw / decode_wire(ApiTran))
def bswap16(x):
    x = np.asarray(x, dtype=np.uint16)
    return ((x >> np.uint16(8)) | (x << np.uint16(8))).astype(np.uint16)


def route_key_ipv4(rec):
    """tcp_ipv4_resp_event_t: (client ip << 32) | client port (the port in network byte order on the wire)"""
    return (rec["daddr"].astype(np.uint64) << np.uint64(32)) | bswap16(rec["dport"]).astype(np.uint64)


def fold_ip6(w):
    """an IPv6 address (4 words) folded to 32 bits: jhash_2words(w2, w3, jhash_2words(w0, w1, GY_SEED))"""
    w = np.asarray(w, dtype=np.uint32)
    return jhash_2words(w[:, 2], w[:, 3], jhash_2words(w[:, 0], w[:, 1], GY_SEED))


def route_key_ipv6(rec):
    return (fold_ip6(rec["daddr"]).astype(np.uint64) << np.uint64(32)) | bswap16(rec["dport"]).astype(np.uint64)


def route_key_resp16(rec):
    """gysk_resp16: the client port alone"""
    return rec["cli_port"].astype(np.uint64)


def route_key_api_tran(rec):
    """API_TRAN: cliport_ alone"""
    return rec["cliport"].astype(np.uint64)


def resp_usec_raw(rec):
    """tresp = lsndtime - lrcvtime msec, kept when <= 1 000 000, as usec"""
    ms = (rec["lsndtime"] - rec["lrcvtime"]).astype(np.uint32)
    return ms, ms <= 1_000_000
