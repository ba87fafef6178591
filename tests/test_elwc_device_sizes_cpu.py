"""PREDICT_ELWCS requests whose list sizes are in device memory (b200tfs_example_device_lists): the C ABI's host arithmetic, no
kernel.  Every argument refusal (on the arena size and on the encode, which checks its arguments before it needs a device), the
closed-form request size refusing device sizes, and the arena bound: the slot of a request with device sizes over a capacity of
N rows holds the request of any sizes adding up to at most N.  The device pointers here are never read."""
import ctypes as C

import numpy as np
import pytest

from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn, RaggedColumn, _example_columns
from min_tfs_client.requests import make_predict_elwcs_request

FAKE_DEV = 0x7F0000001000          # a device address: only compared with NULL and checked for alignment


def _arr(t, v):
    return (t * max(len(v), 1))(*v) if v else None


def _call(input_dict, context_dict, q, n, *, host_sizes=None, dev=FAKE_DEV, kind=N.EXAMPLES_PREDICT_ELWCS):
    """One PREDICT_ELWCS request over the n rows of input_dict with q queries: (structs..., keep-alive)"""
    _, preps = _example_columns(input_dict)
    _, cpreps = _example_columns(context_dict) if context_dict else (0, [])
    feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
    cfeats = (N.Feature * max(len(cpreps), 1))(*[p[0] for p in cpreps])
    req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=3, n_examples=n,
                           n_features=len(preps), flags=0, features=feats)
    tg = N.ExampleTarget(kind=kind, key=b"q", key_len=1)
    hs = None if host_sizes is None else np.ascontiguousarray(host_sizes, np.int64)
    ls = N.ExampleLists(list_sizes=hs.ctypes.data if hs is not None and hs.size else None, n_lists=q, context=cfeats,
                        n_context=len(cpreps), present=1)
    dl = N.ExampleDeviceLists(sizes=dev)
    bs = [p.bytes_entry or N.Bytes() for p in preps]
    rg = [p[3] or N.Ragged() for p in preps]
    lbs = [p.bytes_entry or N.Bytes() for p in cpreps]
    lrg = [p[3] or N.Ragged() for p in cpreps]
    return dict(req=req, tg=tg, ls=ls, dl=dl, bs=bs, rg=rg, lbs=lbs, lrg=lrg, keep=(preps, cpreps, feats, cfeats, hs))


def _arena(lib, s, device=True):
    cap = C.c_uint64()
    rg = _arr(N.Ragged, s["rg"]) if any(g.lengths for g in s["rg"]) else None
    bs = _arr(N.Bytes, s["bs"]) if any(b.offsets for b in s["bs"]) else None
    lrg = _arr(N.Ragged, s["lrg"]) if any(g.lengths for g in s["lrg"]) else None
    lbs = _arr(N.Bytes, s["lbs"]) if any(b.offsets for b in s["lbs"]) else None
    if device:
        rc = lib.b200tfs_example_device_lists_arena_size(1, C.byref(s["req"]), rg, bs, C.byref(s["tg"]), None, None, None, None, None,
                                                         C.byref(s["ls"]), lrg, lbs, C.byref(s["dl"]), C.byref(cap))
    else:
        rc = lib.b200tfs_example_lists_arena_size(1, C.byref(s["req"]), rg, bs, C.byref(s["tg"]), None, None, None, None, None,
                                                  C.byref(s["ls"]), lrg, lbs, C.byref(cap))
    return rc, cap.value


def _encode_args_rc(lib, reqs, tgs, lss, dls):
    """The encode's argument checks, which run before it looks at its (NULL) context"""
    n = len(reqs)
    return lib.b200tfs_encode_example_device_lists_async(None, n, _arr(N.ExampleRequest, reqs), None, None, _arr(N.ExampleTarget, tgs),
                                                         None, None, None, None, None, _arr(N.ExampleLists, lss), None, None,
                                                         _arr(N.ExampleDeviceLists, dls), None, 0)


X = {"x": np.zeros((5, 2), np.float32)}
CD = {"u": np.zeros((3, 1), np.float32)}


def test_device_sizes_accepted_with_any_capacity():
    lib = N.load()
    for n in (0, 1, 5):
        s = _call({"x": np.zeros((n, 2), np.float32)}, CD, 3, n)
        assert _arena(lib, s)[0] == N.OK
    s = _call(X, {}, 0, 5)                       # Q = 0: no size is read, every row goes unsent
    assert _arena(lib, s)[0] == N.OK


def test_refusals():
    lib = N.load()
    ok = _call(X, CD, 3, 5)
    assert _arena(lib, ok)[0] == N.OK
    # device sizes beside host list_sizes on the same request
    both = _call(X, CD, 3, 5, host_sizes=[1, 2, 2])
    assert _arena(lib, both)[0] == N.E_ARG
    assert _encode_args_rc(lib, [both["req"]], [both["tg"]], [both["ls"]], [both["dl"]]) == N.E_ARG
    # neither host nor device sizes with Q > 0
    none = _call(X, CD, 3, 5, dev=None)
    assert _arena(lib, none)[0] == N.E_ARG
    assert _encode_args_rc(lib, [none["req"]], [none["tg"]], [none["ls"]], [none["dl"]]) == N.E_ARG
    # a misaligned device pointer
    mis = _call(X, CD, 3, 5, dev=FAKE_DEV + 4)
    assert _arena(lib, mis)[0] == N.E_ARG
    # a device entry on a request that is not PREDICT_ELWCS, in a call beside a good one
    other = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=0, order=N.ORDER_UPB, version=0, n_examples=0,
                             n_features=0, flags=0, features=None)
    tg_list = N.ExampleTarget(kind=N.EXAMPLES_LIST, key=None, key_len=0)
    no_lists = N.ExampleLists(present=0)
    for dl_other in (N.ExampleDeviceLists(sizes=FAKE_DEV),):
        rc = _encode_args_rc(lib, [ok["req"], other], [ok["tg"], tg_list], [ok["ls"], no_lists], [ok["dl"], dl_other])
        assert rc == N.E_ARG
        cap = C.c_uint64()
        rc = lib.b200tfs_example_device_lists_arena_size(2, _arr(N.ExampleRequest, [ok["req"], other]), None, None,
                                                         _arr(N.ExampleTarget, [ok["tg"], tg_list]), None, None, None, None, None,
                                                         _arr(N.ExampleLists, [ok["ls"], no_lists]), None, None,
                                                         _arr(N.ExampleDeviceLists, [ok["dl"], dl_other]), C.byref(cap))
        assert rc == N.E_ARG
    # ... and with a NULL entry there, the call is accepted
    cap = C.c_uint64()
    rc = lib.b200tfs_example_device_lists_arena_size(2, _arr(N.ExampleRequest, [ok["req"], other]), None, None,
                                                     _arr(N.ExampleTarget, [ok["tg"], tg_list]), None, None, None, None, None,
                                                     _arr(N.ExampleLists, [ok["ls"], no_lists]), None, None,
                                                     _arr(N.ExampleDeviceLists, [ok["dl"], N.ExampleDeviceLists()]), C.byref(cap))
    assert rc == N.OK
    # a device entry on a request whose lists entry is absent (no PREDICT_ELWCS kind)
    s = _call(X, CD, 3, 5, kind=N.EXAMPLES_PREDICT_STRING)
    s["ls"].present = 0
    assert _arena(lib, s)[0] == N.E_ARG
    # the lists-only entry points still refuse NULL host sizes with Q > 0
    assert _arena(lib, ok, device=False)[0] == N.E_ARG


def test_closed_form_size_refuses_device_sizes():
    lib = N.load()
    s = _call(X, CD, 3, 5)
    size = C.c_uint64()
    rc = lib.b200tfs_example_device_lists_request_size(C.byref(s["req"]), C.byref(s["tg"]), None, None, None, None, None,
                                                       C.byref(s["ls"]), None, C.byref(s["dl"]), C.byref(size))
    assert rc == N.E_ARG and "device_lists_arena_size" in N.last_error()
    # with host sizes the new entry point is the lists one
    h = _call(X, CD, 3, 5, host_sizes=[2, 0, 3], dev=None)
    size2 = C.c_uint64()
    assert lib.b200tfs_example_device_lists_request_size(C.byref(h["req"]), C.byref(h["tg"]), None, None, None, None, None,
                                                         C.byref(h["ls"]), None, C.byref(h["dl"]), C.byref(size)) == N.OK
    assert lib.b200tfs_example_lists_request_size(C.byref(h["req"]), C.byref(h["tg"]), None, None, None, None, None,
                                                  C.byref(h["ls"]), None, C.byref(size2)) == N.OK
    want = make_predict_elwcs_request("m", 3, CD, X, [2, 0, 3], "q").ByteSize()
    assert size.value == size2.value == want


def _columns(kind, n, q, rng):
    if kind == "dense":
        return {"x": rng.standard_normal((n, 6)).astype(np.float32)}, {"u": np.ones((q, 40), np.float32)}
    if kind == "int":
        return {"ids": rng.integers(-(1 << 62), 1 << 62, (n, 3))}, {"i": np.full((q, 5), -1, np.int64)}
    if kind == "ragged":
        vals = rng.integers(-(1 << 40), 1 << 40, (n, 4))
        return {"ids": RaggedColumn(vals, rng.integers(0, 5, n))}, {}
    strs = np.array([bytes(rng.integers(97, 123, int(k), dtype=np.uint8)) for k in rng.integers(0, 30, n)], object).astype("S30")
    cstr = np.array([b"c" * int(k) for k in rng.integers(0, 200, q)], object).astype("S200")
    return {"s": BytesColumn.from_array(strs)}, {"t": BytesColumn.from_array(cstr)}


@pytest.mark.parametrize("kind", ["dense", "int", "ragged", "bytes"])
def test_device_arena_bound_holds_any_sizes(kind):
    """For random size vectors of the same Q adding up to at most N, the device-sizes arena (which never reads them) is at least
    the host-sizes arena of those sizes over the first sum(sizes) rows, and at least the request's protobuf size."""
    lib = N.load()
    rng = np.random.default_rng(7)
    for trial in range(12):
        q = int(rng.integers(0, 40))
        n = int(rng.integers(0, 300))
        d, cd = _columns(kind, n, q, rng)
        s_dev = _call(d, cd, q, n)
        rc, dev_cap = _arena(lib, s_dev)
        assert rc == N.OK
        for _ in range(4):
            if q:
                cut = np.sort(rng.integers(0, n + 1, q - 1)) if q > 1 else np.zeros(0, np.int64)
                total = int(rng.integers(cut[-1] if cut.size else 0, n + 1))
                sizes = np.diff(np.concatenate([[0], cut, [total]])).astype(np.int64)
            else:
                sizes, total = np.zeros(0, np.int64), 0
            assert sizes.sum() <= n and (sizes >= 0).all()
            head = {k: _head(v, total) for k, v in d.items()}
            s_host = _call(head, cd, q, total, host_sizes=sizes, dev=None)
            rc, host_cap = _arena(lib, s_host, device=False)
            assert rc == N.OK
            assert dev_cap >= host_cap
            assert dev_cap >= make_predict_elwcs_request("m", 3, cd, head, sizes, "q").ByteSize()


def _head(v, m):
    from min_tfs_client.codec import _head_rows

    return _head_rows(v, m)
