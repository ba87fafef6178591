"""The host side of the padded string decode (b200tfs_padded_strings_layout and the b200tfs_padded_strings mirror) against the
header and the protobuf runtime, on generated ragged responses and on every decode_mutants seed and mutant.  CPU only."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
from google.protobuf.message import DecodeError

import decode_mutants as D
import golden_util as G
import padded_string_decode_ref as PR
import string_responses as SR
from min_tfs_client import _native as N
from tensorflow_serving.apis import predict_pb2

HERE = os.path.dirname(os.path.abspath(__file__))
FIELDS = ("data", "data_cap", "pad", "pad_len", "strings", "data_bytes")


def test_struct_mirror_matches_the_header(tmp_path):
    cc = os.environ.get("CC") or shutil.which("cc") or shutil.which("gcc")
    src = tmp_path / "m.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200tfs.h"\nint main(void) {\n'
                   '  printf("%zu", sizeof(b200tfs_padded_strings));\n'
                   + "".join(f'  printf(" %zu", offsetof(b200tfs_padded_strings, {f}));\n' for f in FIELDS) + "  return 0;\n}\n")
    exe = tmp_path / "m"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(HERE, "..", "include"), "-o", str(exe), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(N.PaddedStrings)] + [getattr(N.PaddedStrings, f).offset for f in FIELDS]


def layout(wires, keys):
    lib = N.load()
    offs = np.cumsum([0] + [len(w) for w in wires[:-1]]).astype(np.uint64)
    n, nk = len(wires), len(keys)
    pk, ps = (N.PadKey * nk)(), (N.PaddedStrings * nk)()
    kb = [k.encode() for k in keys]
    for i, k in enumerate(kb):
        pk[i].key, pk[i].key_len = k, len(k)
    N.check(lib.b200tfs_padded_strings_layout(C.c_char_p(b"".join(wires)), n, (C.c_uint64 * n)(*offs.tolist()),
                                              (C.c_uint64 * n)(*[len(w) for w in wires]), nk, pk, ps, 0))
    return pk, ps


def check_layout(pk, want, what=""):
    """The layout of one string key against the definition's column (want: its tuple or exception type)."""
    if isinstance(want, tuple):
        data, offsets, shape, _ = want
        assert pk.status in (N.OK, N.E_NONCANONICAL), (what, pk.status)
        if pk.status == N.OK:
            assert (pk.dtype, pk.rank) == (SR.DT_STRING, len(shape)), what
            assert tuple(pk.dims[d] for d in range(pk.rank)) == shape, what
            assert pk.bytes == 8 * len(offsets), what
    else:
        assert pk.status != N.OK or pk.dtype != SR.DT_STRING, (what, want)


def own_strings(wires, key):
    S = [s for w in wires for s in predict_pb2.PredictResponse.FromString(w).outputs[key].string_val]
    return len(S), sum(len(s) for s in S)


def test_layout_on_ragged_responses():
    rng = np.random.default_rng(11)
    wires = []
    for r in range(12):
        t, k = int(rng.integers(0, 6)), int(rng.integers(1, 4))
        wires.append(SR.response(("f", SR.float_tensor(np.ones((1, t, 3), np.float32))),
                                 ("s", SR.string_tensor(SR.random_strings(rng, t * k, 0, 200), [t, k]))))
    pk, ps = layout(wires, ["s", "f"])
    want = PR.reference(wires, "s")
    check_layout(pk[0], want)
    assert pk[0].status == N.OK
    assert (ps[0].strings, ps[0].data_bytes) == own_strings(wires, "s")
    assert (pk[1].status, pk[1].dims[1], ps[1].strings, ps[1].data_bytes) == (N.OK, 5, 0, 0)
    assert pk[1].bytes == 4 * 3 * 5 * 12
    # without entries: today's layout, a string key OK with no bytes
    lib = N.load()
    pk2 = (N.PadKey * 1)()
    pk2[0].key, pk2[0].key_len = b"s", 1
    offs = np.cumsum([0] + [len(w) for w in wires[:-1]]).astype(np.uint64)
    N.check(lib.b200tfs_padded_layout(C.c_char_p(b"".join(wires)), 12, (C.c_uint64 * 12)(*offs.tolist()),
                                      (C.c_uint64 * 12)(*[len(w) for w in wires]), 1, pk2, 0))
    assert (pk2[0].status, pk2[0].bytes, pk2[0].dims[0]) == (N.OK, 0, pk[0].dims[0])


def test_layout_statuses():
    s = [b"a", b"bc"]
    good = SR.response(("s", SR.string_tensor(s, [2])))
    assert layout([good, SR.response(("t", SR.string_tensor(s, [2])))], ["s"])[0][0].status == N.E_KEY
    assert layout([good, SR.response(("s", SR.string_tensor(s, [1, 2])))], ["s"])[0][0].status == N.E_SHAPE
    assert layout([good, SR.response(("s", SR.string_tensor(s, [])))], ["s"])[0][0].status == N.E_SHAPE
    assert layout([good, SR.response(("s", SR.string_tensor(s, [3])))], ["s"])[0][0].status == N.E_SHAPE
    assert layout([good, SR.response(("s", SR.float_tensor(np.ones(2, np.float32))))], ["s"])[0][0].status == N.E_DTYPE
    assert layout([good, good[:-3]], ["s"])[0][0].status == N.E_PARSE
    s8 = SR.random_strings(np.random.default_rng(1), 8, 1, 5)
    merged = G.ld(0x0A, G.ld(0x0A, b"s") + G.ld(0x12, SR.string_tensor(s8[:4], [8])) + G.ld(0x12, SR.strings_body(s8[4:]))) + G.mspec()
    pk, ps = layout([good, merged], ["s"])
    assert (pk[0].status, pk[0].bad_rec, ps[0].strings) == (N.E_NONCANONICAL, 1, 0)


def test_layout_on_every_mutant():
    checked = 0
    for seed, ms in D.corpus():
        if seed.tensor:
            continue
        keys = [k for k, t in predict_pb2.PredictResponse.FromString(seed.wire).outputs.items() if t.dtype == SR.DT_STRING]
        for m in [D.Mutant(seed.name, "seed", seed.wire, len(seed.wire))] + ms:
            rec = m.record
            for key in keys:
                want = SR.outcome(lambda: PR.reference([rec], key))
                pk, ps = layout([rec], [key])
                if want is DecodeError and pk[0].status == N.OK:
                    continue      # malformed varints of an unrequested output: the decode reads only the requested one
                check_layout(pk[0], want, (seed.name, m.kind, m.rec_len))
                if isinstance(want, tuple) and pk[0].status == N.OK:
                    assert (ps[0].strings, ps[0].data_bytes) == own_strings([rec], key), (seed.name, m.kind)
                    checked += 1
    assert checked > 10
