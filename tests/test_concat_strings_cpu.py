"""The string_val walk of the concatenated string decode (csrc/string_walk.h) and its host layout, against the protobuf runtime.

CPU only: the walk compiled for the host (tests/native/string_walk_host.cpp), composed as str_index_kernel composes it, must find
exactly the strings PredictResponse.FromString gives - on generated responses and on every decode_mutants seed and mutant - and
b200tfs_concat_strings_layout must report the counts, bytes and statuses of the definition (tests/string_responses.py).  The GPU
test runs the same cases through the kernels.
"""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
from google.protobuf.message import DecodeError

import decode_mutants as D
import golden_util as G
import string_responses as SR
from min_tfs_client import _native as N
from tensorflow_serving.apis import predict_pb2

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = os.environ.get("CXX") or shutil.which("g++") or "c++"
    so = str(tmp_path_factory.mktemp("sw") / "libstring_walk_host.so")
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unknown-pragmas", "-shared", "-o", so,
                    os.path.join(HERE, "native", "string_walk_host.cpp")], check=True)
    L = C.CDLL(so)
    L.sw_strings.restype = C.c_int
    L.sw_strings.argtypes = [C.c_char_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    L.sw_count_bound.restype = C.c_uint64
    L.sw_count_bound.argtypes = [C.c_uint64]
    return L


def walk_strings(lib, rec: bytes, o: N.Output):
    cap = max(len(rec) // 2, 1)
    off, ln, cnt = np.zeros(cap, np.uint64), np.zeros(cap, np.uint32), C.c_uint64()
    st = lib.sw_strings(rec, len(rec), o.msg_off, o.msg_len, off.ctypes.data, ln.ctypes.data, cap, C.byref(cnt))
    n = cnt.value
    return st, [rec[int(off[j]): int(off[j]) + int(ln[j])] for j in range(min(n, cap))], n


def check_record(lib, buf: bytes, rec_len: int, what=""):
    """Every DT_STRING output the host walker tabulates: the string walk against the runtime.  Returns how many it walked."""
    rec = bytes(buf[:rec_len])
    w = D.walk(buf, rec_len)
    if w.status != N.OK:
        return 0
    try:
        parsed = predict_pb2.PredictResponse.FromString(rec)
    except DecodeError:
        return 0          # a packed-varint payload malformed inside: not the string walk's concern
    walked = 0
    for o in w.outs:
        if o.dtype != SR.DT_STRING or o.status != N.OK:
            continue
        key = rec[o.key_off: o.key_off + o.key_len].decode()
        want = list(parsed.outputs[key].string_val)
        st, got, n = walk_strings(lib, rec, o)
        assert st == N.OK, (what, key, st)
        assert len(want) == o.n_strings, (what, key)
        if n == o.n_strings:
            assert got == want, (what, key)
        else:             # the TensorProto in several `value` occurrences: the last one holds fewer (the device route refuses)
            assert n < o.n_strings and got == want[len(want) - n:], (what, key)
        walked += 1
    return walked


def cases():
    rng = np.random.default_rng(7)
    edge = [b"", b"\x00", b"\x00\xff\x80", b"x" * 127, b"y" * 128, b"z" * 16383, b"w" * 16384, b"\xfe" * 70000]
    s = SR.random_strings(rng, 12, 0, 40)
    return {
        "edges": SR.response(("s", SR.string_tensor(edge, [len(edge)]))),
        "empty": SR.response(("s", SR.string_tensor([b""] * 5, [5, 1]))),
        "zero_rows": SR.response(("s", SR.string_tensor([], [0, 3]))),
        "infer": SR.response(("s", SR.string_tensor(s, [-1, 3]))),
        "dtype_last": SR.response(("s", SR.string_tensor(s, [4, 3], dtype_last=True))),
        "unknown": SR.response(("s", SR.string_tensor(s, [12], unknown=True))),
        "mixed": SR.response(("f", SR.float_tensor(np.ones((2, 3), np.float32))), ("s", SR.string_tensor(s[:6], [2, 3])),
                             ("i", SR.int64_tensor(np.arange(6).reshape(2, 3))), ("t", SR.string_tensor(s[6:], [6]))),
        # one map entry whose TensorProto arrives in two `value` occurrences: the runtime merges them
        "merged": merged_response(s),
    }


def merged_response(s):
    first = G.ld(0x12, SR.string_tensor(s[:4], [8]))
    second = G.ld(0x12, SR.strings_body(s[4:8]))
    return G.ld(0x0A, G.ld(0x0A, b"s") + first + second) + G.mspec()


@pytest.mark.parametrize("name", list(cases()))
def test_walk_agrees_with_the_runtime(lib, name):
    w = cases()[name]
    assert check_record(lib, w, len(w), name) == (2 if name == "mixed" else 1)


def test_walk_on_every_mutant(lib):
    walked = 0
    for seed, ms in D.corpus():
        if seed.tensor:
            continue
        walked += check_record(lib, seed.wire, len(seed.wire), seed.name)
        for m in ms:
            walked += check_record(lib, m.buf, m.rec_len, (m.seed, m.kind, m.rec_len))
    assert walked > 100      # the "multi" seed's string output, and its accepted mutants


def layout(wires, keys):
    lib = N.load()
    offs = np.cumsum([0] + [len(w) for w in wires[:-1]]).astype(np.uint64)
    n, nk = len(wires), len(keys)
    ck, sc = (N.ConcatKey * nk)(), (N.ConcatStrings * nk)()
    kb = [k.encode() for k in keys]
    for i, k in enumerate(kb):
        ck[i].key, ck[i].key_len = k, len(k)
    N.check(lib.b200tfs_concat_strings_layout(C.c_char_p(b"".join(wires)), n, (C.c_uint64 * n)(*offs.tolist()),
                                              (C.c_uint64 * n)(*[len(w) for w in wires]), nk, ck, sc, 0))
    return ck, sc


def test_layout_counts_bytes_and_shape():
    rng = np.random.default_rng(3)
    wires = []
    for r in range(9):
        s = SR.random_strings(rng, 5 * (r % 4), 0, 300)
        wires.append(SR.response(("f", SR.float_tensor(np.ones((r % 4, 5), np.float32))), ("s", SR.string_tensor(s, [r % 4, 5]))))
    ck, sc = layout(wires, ["s", "f"])
    data, offsets, shape = SR.reference(wires, "s")
    assert (ck[0].status, ck[0].dtype, ck[0].rank) == (N.OK, SR.DT_STRING, 2)
    assert (ck[0].dims[0], ck[0].dims[1]) == shape
    assert (sc[0].strings, sc[0].data_bytes, ck[0].bytes) == (len(offsets) - 1, len(data), 8 * len(offsets))
    assert (ck[1].status, ck[1].bytes, sc[1].strings, sc[1].data_bytes) == (N.OK, 4 * 5 * sum(r % 4 for r in range(9)), 0, 0)


def test_layout_statuses():
    s = [b"a", b"bc"]
    good = SR.response(("s", SR.string_tensor(s, [2])))
    assert layout([good, SR.response(("t", SR.string_tensor(s, [2])))], ["s"])[0][0].status == N.E_KEY
    assert layout([good, SR.response(("s", SR.string_tensor(s, [1, 2])))], ["s"])[0][0].status == N.E_SHAPE
    assert layout([good, SR.response(("s", SR.string_tensor(s, [])))], ["s"])[0][0].status == N.E_SHAPE
    assert layout([good, SR.response(("s", SR.string_tensor(s, [3])))], ["s"])[0][0].status == N.E_SHAPE
    assert layout([good, SR.response(("s", SR.float_tensor(np.ones(2, np.float32))))], ["s"])[0][0].status == N.E_DTYPE
    assert layout([good, good[:-3]], ["s"])[0][0].status == N.E_PARSE
    ck, sc = layout([good, merged_response(SR.random_strings(np.random.default_rng(1), 8, 1, 5))], ["s"])
    assert (ck[0].status, ck[0].bad_rec, sc[0].strings) == (N.E_NONCANONICAL, 1, 0)


def test_struct_mirror_and_bound(lib):
    assert C.sizeof(N.ConcatStrings) == 32
    assert [getattr(N.ConcatStrings, f).offset for f in ("data", "data_cap", "strings", "data_bytes")] == [0, 8, 16, 24]
    lens = [0, 1, 2, 3, 1000, 12345]
    ms, mb = C.c_uint64(), C.c_uint64()
    N.check(N.load().b200tfs_concat_strings_bound(len(lens), (C.c_uint64 * len(lens))(*lens), C.byref(ms), C.byref(mb)))
    assert (ms.value, mb.value) == (sum(x // 2 for x in lens), sum(lens))
    assert all(lib.sw_count_bound(x) == x // 2 for x in lens)
    # a response of nothing but empty strings comes close: the bound holds and is tight to the framing
    for n in (1, 100, 5000):
        w = SR.response(("s", SR.string_tensor([b""] * n, [n])), spec=False)
        ck, sc = layout([w], ["s"])
        N.check(N.load().b200tfs_concat_strings_bound(1, (C.c_uint64 * 1)(len(w)), C.byref(ms), C.byref(mb)))
        assert sc[0].strings == n <= ms.value < n + 16 and sc[0].data_bytes <= mb.value
