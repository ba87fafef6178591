"""b200tfs_decode_slot_bytes: the slot the single-launch decode lays out for host-resident records, computed without a device."""
import ctypes as C

import numpy as np

import decode_mutants as D
from min_tfs_client import _native as N


def fld(field, payload):
    return D.vi((field << 3) | 2) + D.vi(len(payload)) + payload


def resp(*outs):
    return b"".join(D.entry(k, D.tproto(dt, dims, fld(field, body))) for k, dt, dims, field, body in outs) + D.mspec()


def slot(recs, varints):
    lib = N.load()
    buf = b"".join(recs)
    offs, cur = [], 0
    for r in recs:
        offs.append(cur)
        cur += len(r)
    n = len(recs)
    need, nv = C.c_uint64(), C.c_int32()
    N.check(lib.b200tfs_decode_slot_bytes(C.c_char_p(buf), n, (C.c_uint64 * n)(*offs), (C.c_uint64 * n)(*[len(r) for r in recs]),
                                          varints, C.byref(need), C.byref(nv)))
    return need.value, nv.value


def test_varint_ranges_in_table_order_and_the_most_any_record_needs():
    ids = b"".join(D.vi(v) for v in range(200))
    f = np.zeros(64, np.float32).tobytes()
    a = resp(("ids", 9, [200], 10, ids), ("f", 1, [64], 5, f))          # int64[200] (1600 B) first, then 256 B of floats
    b = resp(("f", 1, [64], 5, f), ("m", 10, [3], 11, b"\x01\x00\x01"))  # floats first, then bool[3]
    assert slot([a], 1) == (1792 + 256, 1)
    assert slot([a], 0) == (256, 0)                                      # switch off: the floats alone, at offset 0
    assert slot([b], 1) == (256 + 3, 1)
    assert slot([b, a], 1) == (2048, 2)
    # a denser response of the same model needs more than its wire length suggests: 4096 zeros take 1 wire byte and 8 slot bytes each
    dense = resp(("ids", 9, [4096], 10, b"\x00" * 4096), ("f", 1, [64], 5, f))
    assert slot([dense], 1) == (32768 + 256, 1)


def test_records_that_do_not_walk_need_nothing():
    ok = resp(("ids", 9, [2], 10, b"\x01\x02"))
    assert slot([ok[:-3]], 1) == (0, 0)
    assert slot([ok[:-3], ok], 1) == (16, 1)
