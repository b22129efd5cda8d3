"""The record layouts the decoders read, pinned to the reference's own struct definitions (CPU only).

tests/golden/wire_ref_golden.npz holds the sizes, alignments and field offsets of the reference's COMM_HEADER, EVENT_NOTIFY,
TCP_CONN_NOTIFY, AGGR_TASK_STATE_NOTIFY, LISTENER_STATE_NOTIFY, HOST_STATE_NOTIFY, ACTIVE_CONN_STATS, LISTENER_DAY_STATS,
AGGR_TASK_HIST_STATS, API_TRAN and the four eBPF records, as compiled from the reference tree (oracle/ref_wire.cc), and records the
reference wrote from seeded field values. Here every mirror is held to it:
  - the C++ structs of gyeeta_b200/csrc/gysk_wire.h (offsetof / sizeof / alignof printed by a small compiled program), and the
    API_TRAN_OFF constants with the widths gysk_engine.cu reads at them;
  - the numpy dtypes of gyeeta_b200/wire.py, and its encoders given the same field values (bytes equal, padding zero on both sides);
  - the shim's size checks of the eBPF records.
When oracle/_ref/libgyrefwire.so is present, the fixture is rebuilt from it and must equal the file."""
import os
import re
import subprocess

import numpy as np
import pytest

from gyeeta_b200 import wire
from oracle import pyoracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "wire_ref_golden.npz")

# reference struct -> gysk_wire.h mirror (None: checked through API_TRAN_OFF); reference field -> mirror member where they differ
HDR_STRUCT = {"GY_IP_ADDR": "IP_PORT", "API_TRAN": None}
HDR_FIELD = {("tcp_ipv4_resp_event_t", "tup.saddr"): "saddr", ("tcp_ipv4_resp_event_t", "tup.daddr"): "daddr",
             ("tcp_ipv4_resp_event_t", "tup.netns"): "netns", ("tcp_ipv4_resp_event_t", "tup.sport"): "sport",
             ("tcp_ipv4_resp_event_t", "tup.dport"): "dport", ("tcp_ipv6_resp_event_t", "tup.saddr"): "saddr",
             ("tcp_ipv6_resp_event_t", "tup.daddr"): "daddr", ("tcp_ipv6_resp_event_t", "tup.netns"): "netns",
             ("tcp_ipv6_resp_event_t", "tup.sport"): "sport", ("tcp_ipv6_resp_event_t", "tup.dport"): "dport"}
# fields the mirror does not spell out (GY_IP_ADDR is restated flat inside IP_PORT; its members are checked one by one)
HDR_SKIP = {("IP_PORT", "ipaddr_")}
# the API_TRAN fields the decoders read, by API_TRAN_OFF constant
API_OFF = dict(TUPD_USEC="tupd_usec_", REQLEN="reqlen_", RESLEN="reslen_", REQNUM="reqnum_", RESPONSE_USEC="response_usec_",
               GLOB_ID="glob_id_", ERRORCODE="errorcode_", CLIPORT="cliport_", REQUEST_LEN="request_len_", LENEXT="lenext_", PADLEN="padlen_")

# reference struct -> (wire.py dtype, {reference field: dtype field}); fields not listed are the reference's name without its trailing _
RENAME = {"cli_ser_machine_id_": "machid", "remote_machine_id_": "machid", "is_tcp_connect_event_": "is_connect",
          "is_tcp_accept_event_": "is_accept", "is_loopback_conn_": "is_loopback", "ip128_be_": "ip128", "ip32_be_": "ip32",
          "cliip_": "cliip", "serip_": "serip"}
PY = {"IP_PORT": wire.IP_PORT, "TCP_CONN_NOTIFY": wire.TCP_CONN, "AGGR_TASK_STATE_NOTIFY": wire.TASK,
      "AGGR_TASK_HIST_STATS": wire.AGGR_TASK_HIST_STATS, "ACTIVE_CONN_STATS": wire.ACTIVE, "API_TRAN": wire.API_TRAN,
      "tcp_ipv4_event_t": wire.CONN4, "tcp_ipv6_event_t": wire.CONN6, "tcp_ipv4_resp_event_t": wire.RESP4, "tcp_ipv6_resp_event_t": wire.RESP6}
PY_SKIP = {("IP_PORT", "ipaddr_")}


def py_field(strct, field):
    return RENAME.get(field, field.split(".")[-1].rstrip("_"))


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def table(g):
    structs = {str(n): (int(s), int(a)) for n, s, a in zip(g["layout_struct_name"], g["layout_struct_size"], g["layout_struct_align"])}
    fields = [(str(t), str(f), int(o), int(s)) for t, f, o, s in zip(g["layout_field_struct"], g["layout_field_name"], g["layout_field_off"],
                                                                    g["layout_field_size"])]
    return structs, fields


@pytest.fixture(scope="module")
def mirror(g, tmp_path_factory):
    """what the compiler makes of gysk_wire.h: {(struct, member): (offset, size)}, {(struct, "sizeof"/"alignof"): n}"""
    structs, fields = table(g)
    lines = []
    for t in structs:
        if t not in ("GY_IP_ADDR", "API_TRAN"):
            lines.append(f"S({t})")
    for t, f, _, _ in fields:
        m = HDR_STRUCT.get(t, t)
        mf = HDR_FIELD.get((t, f), f)
        if m and (m, mf) not in HDR_SKIP:
            lines.append(f"F({m}, {mf})")
    for k in API_OFF:
        lines.append(f'std::printf("API_TRAN_OFF {k} %zu 0\\n", (size_t)API_TRAN_OFF::{k});')
    lines.append('std::printf("API_TRAN_OFF SIZE %zu 0\\n", (size_t)API_TRAN_OFF::SIZE);')
    src = ("#include <cstddef>\n#include <cstdio>\n#include \"gysk_wire.h\"\nusing namespace gysk::wire;\n"
           "#define F(T, f) std::printf(#T \" \" #f \" %zu %zu\\n\", offsetof(T, f), sizeof(((T *)0)->f));\n"
           "#define S(T) std::printf(#T \" sizeof %zu 0\\n\" #T \" alignof %zu 0\\n\", sizeof(T), alignof(T));\n"
           "int main()\n{\n" + "\n".join(lines) + "\nreturn 0;\n}\n")
    d = tmp_path_factory.mktemp("wire_layout")
    cc, exe = os.path.join(str(d), "layout.cc"), os.path.join(str(d), "layout")
    with open(cc, "w") as fh:
        fh.write(src)
    subprocess.run(["g++", "-std=c++17", "-O0", "-w", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "gyeeta_b200", "csrc"),
                    cc, "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split("\n")
    return {(t, f): (int(o), int(s)) for t, f, o, s in (line.split() for line in out if line)}


def test_fixture_covers_every_struct_the_decoders_read(g):
    structs, fields = table(g)
    assert set(structs) == {"COMM_HEADER", "EVENT_NOTIFY", "GY_IP_ADDR", "IP_PORT", "TCP_CONN_NOTIFY", "AGGR_TASK_STATE_NOTIFY",
                            "LISTENER_STATE_NOTIFY", "HOST_STATE_NOTIFY", "ACTIVE_CONN_STATS", "LISTENER_DAY_STATS", "AGGR_TASK_HIST_STATS",
                            "API_TRAN", "tcp_ipv4_event_t", "tcp_ipv6_event_t", "tcp_ipv4_resp_event_t", "tcp_ipv6_resp_event_t"}
    named = {(t, f) for t, f, _, _ in fields}
    assert {("API_TRAN", f) for f in API_OFF.values()} <= named
    # each struct's fields are listed in offset order and do not overlap
    for t in structs:
        fs = sorted((o, s, f) for tt, f, o, s in fields if tt == t)
        for (o1, s1, f1), (o2, _, f2) in zip(fs, fs[1:]):
            assert o1 + s1 <= o2 or t == "IP_PORT", f"{t}.{f1} overlaps {t}.{f2}"
        assert fs[-1][0] + fs[-1][1] <= structs[t][0], t


def test_gysk_wire_h_matches_reference(g, mirror):
    structs, fields = table(g)
    for t, (size, align) in structs.items():
        m = HDR_STRUCT.get(t, t)
        if m is None or t == "GY_IP_ADDR":
            continue
        assert mirror[(m, "sizeof")][0] == size, f"gysk_wire.h {m}: sizeof {mirror[(m, 'sizeof')][0]}, reference {t} {size}"
        assert mirror[(m, "alignof")][0] == align, f"gysk_wire.h {m}: alignof {mirror[(m, 'alignof')][0]}, reference {t} {align}"
    for t, f, off, size in fields:
        m = HDR_STRUCT.get(t, t)
        mf = HDR_FIELD.get((t, f), f)
        if m is None or (m, mf) in HDR_SKIP:
            continue
        got = mirror[(m, mf)]                   # GY_IP_ADDR is restated flat at the start of IP_PORT: the same offsets
        assert got == (off, size), f"gysk_wire.h {m}.{mf}: offset/size {got}, reference {t}.{f} {(off, size)}"


def test_api_tran_offsets_match_reference(g, mirror):
    structs, fields = table(g)
    ref = {f: (o, s) for t, f, o, s in fields if t == "API_TRAN"}
    assert mirror[("API_TRAN_OFF", "SIZE")][0] == structs["API_TRAN"][0], "API_TRAN_OFF::SIZE"
    for k, f in API_OFF.items():
        assert mirror[("API_TRAN_OFF", k)][0] == ref[f][0], f"API_TRAN_OFF::{k} = {mirror[('API_TRAN_OFF', k)][0]}, reference API_TRAN.{f} at {ref[f][0]}"
    # the width each decoder reads at a constant is the reference field's width
    src = open(os.path.join(ROOT, "gyeeta_b200", "csrc", "gysk_engine.cu")).read()
    reads = re.findall(r"at<(u?int\d+_t)>\(O::(\w+)\)", src) + [("uint8_t", k) for k in re.findall(r"p\[O::(\w+)\]", src)]
    assert {k for _, k in reads} == set(API_OFF), "every API_TRAN_OFF field is read by a decoder"
    width = {"uint8_t": 1, "uint16_t": 2, "int32_t": 4, "uint32_t": 4, "uint64_t": 8}
    for ty, k in reads:
        assert width[ty] == ref[API_OFF[k]][1], f"decoder reads API_TRAN_OFF::{k} as {ty}, reference API_TRAN.{API_OFF[k]} is {ref[API_OFF[k]][1]} bytes"
    assert ("int32_t", "ERRORCODE") in reads                              # errorcode_ is a signed int in the reference


def test_wire_py_dtypes_match_reference(g):
    structs, fields = table(g)
    for t, dt in PY.items():
        assert dt.itemsize == structs[t][0], f"wire.py {t}: itemsize {dt.itemsize}, reference {structs[t][0]}"
    for t, f, off, size in fields:
        dt = PY.get("IP_PORT" if t == "GY_IP_ADDR" else t)
        if dt is None or (t, f) in PY_SKIP:
            continue
        pf = py_field(t, f)
        assert pf in dt.names, f"wire.py {t}: no field {pf} for reference {t}.{f}"
        fdt, foff = dt.fields[pf][:2]
        assert (foff, fdt.itemsize) == (off, size), f"wire.py {t}.{pf}: offset/size {(foff, fdt.itemsize)}, reference {t}.{f} {(off, size)}"
    # COMM_HEADER + EVENT_NOTIFY are one dtype in wire.py
    hdr = {f: (o, s) for t, f, o, s in fields if t in ("COMM_HEADER", "EVENT_NOTIFY")}
    base = structs["COMM_HEADER"][0]
    for f, pf, b in (("magic_", "magic", 0), ("total_sz_", "total_sz", 0), ("data_type_", "data_type", 0), ("padding_sz_", "padding_sz", 0),
                     ("subtype_", "subtype", base), ("nevents_", "nevents", base)):
        assert (wire.HDR.fields[pf][1], wire.HDR.fields[pf][0].itemsize) == (b + hdr[f][0], hdr[f][1]), f"wire.py HDR.{pf}"
    assert wire.HDR.itemsize == structs["COMM_HEADER"][0] + structs["EVENT_NOTIFY"][0]


def test_shim_record_sizes_match_reference(g):
    structs, _ = table(g)
    src = open(os.path.join(ROOT, "gyeeta_b200", "host", "gy_gysk_shim.h")).read()
    resp = re.search(r"sizeof\(RespEvent\) == (\d+) \|\| sizeof\(RespEvent\) == (\d+)", src).groups()
    conn = re.search(r"sizeof\(ConnEvent\) == (\d+) \|\| sizeof\(ConnEvent\) == (\d+)", src).groups()
    assert tuple(map(int, resp)) == (structs["tcp_ipv4_resp_event_t"][0], structs["tcp_ipv6_resp_event_t"][0])
    assert tuple(map(int, conn)) == (structs["tcp_ipv4_event_t"][0], structs["tcp_ipv6_event_t"][0])


def sets(g):
    return sorted({k.split("__")[0] for k in g.files if k.endswith("__struct")})


def values(g, name):
    return {str(f): g[f"{name}.{f}"] for f in g[f"{name}__fields"]}


def tails(g, name):
    if f"{name}__tail" not in g.files:
        return None
    t, o = g[f"{name}__tail"].tobytes(), g[f"{name}__toff"]
    return [t[int(a): int(b)] for a, b in zip(o[:-1], o[1:])]


def encode(strct, vals, n):
    """the wire.py records of strct filled from the golden field values"""
    dt = PY[strct]
    rec = np.zeros(n, dtype=dt)
    for f, a in vals.items():
        pf = py_field(strct, f)
        if strct == "ACTIVE_CONN_STATS" and f in ("cli_listener_proc_", "is_remote_listen_", "is_remote_cli_"):
            bit = ("cli_listener_proc_", "is_remote_listen_", "is_remote_cli_").index(f)
            rec["flags"] |= (a.astype(np.uint8) & 1) << bit
            continue
        col = rec[pf]
        if col.dtype.kind == "V" or col.dtype.kind == "S" or col.dtype.subdtype is not None or a.ndim > 1:
            raw = rec.view(np.uint8).reshape(n, -1)
            off, sz = dt.fields[pf][1], dt.fields[pf][0].itemsize
            raw[:, off: off + sz] = np.ascontiguousarray(a).view(np.uint8).reshape(n, -1)
        else:
            rec[pf] = a.view(col.dtype) if a.dtype.itemsize == col.dtype.itemsize and a.dtype.kind != col.dtype.kind else a
    return rec


def test_golden_sets_reach_the_edges(g):
    v = values(g, "tcp_conn")
    assert (v["tusec_close_"] == 0).any() and (v["tusec_close_"] != 0).any()
    assert (v["tusec_start_"] == (1 << 32) * 10 ** 6 - 1).any() and (v["tusec_start_"] > 1.7e15).any()
    s = v["bytes_sent_"].astype(object) + v["bytes_rcvd_"].astype(object)
    assert any(x < 1 << 32 for x in s) and any(x >= 1 << 32 for x in s)
    assert (v["ser_glob_id_"] == 0).any() and (v["cli_task_aggr_id_"] == 0).any()
    a = values(g, "active")
    sh = [(int(x) + int(y)) >> 10 for x, y in zip(a["bytes_sent_"], a["bytes_received_"])]
    assert (1 << 32) - 1 in sh and 1 << 32 in sh and (a["listener_glob_id_"] == 0).any()
    assert (a["max_rtt_msec_"] < 0).any() and (a["max_rtt_msec_"] == 0).any() and (a["max_rtt_msec_"] % 1 != 0).any()
    assert (values(g, "task")["aggr_task_id_"] == 0).any() and (values(g, "task")["total_cpu_pct_"] % 1 != 0).any()
    for name in ("ipv4_event", "ipv6_event"):
        ev = values(g, name)
        assert set(np.unique(ev["type"])) == {0, 1, 2, 3, 4, 5} and (ev["ts_ns"] > 1.7e18).any()
        assert {0, 1, 255, 256, 65535} <= set(ev["sport"].byteswap().tolist())
    for name in ("ipv4_resp", "ipv6_resp"):
        r = values(g, name)
        d = (r["lsndtime"] - r["lrcvtime"]).astype(np.uint32)
        assert {1_000_000, 1_000_001, 0xFFFFFFFF} <= set(d.tolist())
    w = values(g, "ipv6_event")["saddr"].view(np.uint32).reshape(-1, 4)
    assert (w[:, 2] == np.uint32(0xFFFF0000).byteswap()).any() and (w[:, 0] != 0).any()
    t = values(g, "api_tran")
    assert {0, 1, 499, 500} <= set(t["errorcode_"].tolist()) and (t["reqnum_"] == 0).any()
    assert {0, 1, 255, 256, 65535} <= set(t["cliport_"].tolist())
    for name in ("tcp_conn", "task", "listener", "api_tran"):
        lens = [len(x) for x in tails(g, name)]
        assert {0, 1, 7, 8}.issubset(lens) and max(lens) >= 255
    assert len(values(g, "tcp_conn")["tusec_start_"]) == 2048 and len(values(g, "task")["aggr_task_id_"]) == 1200
    assert len(values(g, "listener")["glob_id_"]) == 512 and len(values(g, "active")["listener_glob_id_"]) == 2048
    assert len(values(g, "api_tran")["glob_id_"]) == 256


def walk(buf, fixed, lenfield, padfield, n, extra=None):
    """(record start, fixed part end, element end) of each variable-stride record"""
    out, p = [], 0
    for _ in range(n):
        rec = np.frombuffer(buf[p: p + fixed.itemsize], dtype=fixed)[0]
        es = fixed.itemsize + int(rec[lenfield]) + (int(rec[extra]) if extra else 0) + int(rec[padfield])
        out.append((p, es))
        p += es
    assert p == len(buf)
    return out


@pytest.mark.parametrize("name", ["tcp_conn", "task", "active", "api_tran", "ipv4_event", "ipv6_event", "ipv4_resp", "ipv6_resp"])
def test_wire_py_encoders_equal_reference_bytes(g, name):
    strct = str(g[f"{name}__struct"])
    vals = values(g, name)
    n = len(next(iter(vals.values())))
    rec = encode(strct, vals, n)
    ref = g[f"{name}__bytes"].tobytes()
    tl = tails(g, name)
    if strct in ("TCP_CONN_NOTIFY", "AGGR_TASK_STATE_NOTIFY"):
        msg = bytes(wire.build_msg(int(g[f"{name}__subtype"]), [(rec[i: i + 1], tl[i]) for i in range(n)]))
        want = g[f"{name}__msg_head"].tobytes() + ref + b"\0" * (int(g[f"{name}__msg_len"]) - 24 - len(ref))
        assert msg[:24] == want[:24], f"{strct}: message header differs"
        body = msg[24:]
    elif strct == "API_TRAN":
        body = bytes(wire.pack_api_tran(rec, tl))
    elif strct == "ACTIVE_CONN_STATS":
        msg = wire.build_msg_fixed(int(g[f"{name}__subtype"]), rec).tobytes()
        want = g[f"{name}__msg_head"].tobytes() + ref
        assert msg == want, f"{strct}: message differs"
        body = msg[24:]
    else:
        body = rec.tobytes()
    assert len(body) == len(ref), f"{strct}: {len(body)} bytes, reference {len(ref)}"
    if body != ref:
        a, b = np.frombuffer(body, np.uint8), np.frombuffer(ref, np.uint8)
        i = int(np.flatnonzero(a != b)[0])
        raise AssertionError(f"{strct}: first differing byte {i} (wire.py {a[i]}, reference {b[i]})")


def test_reference_padding_is_zero(g):
    """the reference builders leave every padding byte zero, so the byte-for-byte comparisons cover padding too"""
    for name, fixed, lf, pf, ext in (("tcp_conn", wire.TCP_CONN, "cli_cmdline_len", "padding_len", None),
                                     ("task", wire.TASK, "issue_string_len", "padding_len", None),
                                     ("api_tran", wire.API_TRAN, "request_len", "padlen", "lenext")):
        buf = g[f"{name}__bytes"].tobytes()
        n = len(g[f"{name}__toff"]) - 1
        pads = set()
        for (p, es), t in zip(walk(buf, fixed, lf, pf, n, ext), tails(g, name)):
            rec = np.frombuffer(buf[p: p + fixed.itemsize], dtype=fixed)[0]
            assert es % 8 == 0 and int(rec[lf]) == len(t)
            assert buf[p + fixed.itemsize: p + fixed.itemsize + len(t)] == t
            assert not any(buf[p + fixed.itemsize + len(t): p + es]), name
            pads.add(int(rec[pf]))
        assert pads == set(range(8)), (name, pads)
    # the listener records: every padding length, a zero tail
    buf = g["listener__bytes"].tobytes()
    p, pads = 0, set()
    for t in tails(g, "listener"):
        sl, pl = buf[p + 85], buf[p + 86]
        assert sl == len(t) and buf[p + 88: p + 88 + sl] == t and not any(buf[p + 88 + sl: p + 88 + sl + pl])
        pads.add(pl)
        p += 88 + sl + pl
    assert p == len(buf) and pads == set(range(8))


def test_fixture_is_current():
    """rebuilt from the reference library, the fixture equals the committed file (only where oracle/_ref holds the library)"""
    R = po.refwire()
    if R is None:
        pytest.skip("oracle/_ref/libgyrefwire.so absent (built by oracle/Makefile where the reference tree exists)")
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_wire_golden", os.path.join(ROOT, "tests", "golden", "make_wire_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    fresh = mk.generate(R)
    g = np.load(GOLDEN)
    assert sorted(fresh) == sorted(g.files)
    for k, a in fresh.items():
        assert np.array_equal(np.asarray(a), g[k]), f"{k} differs from the reference: run python tests/golden/make_wire_golden.py"
