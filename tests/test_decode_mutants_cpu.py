"""The mutant corpus (tests/decode_mutants.py) through the host build of the tag walker, against the protobuf runtime and the
reference's algorithm (oracle/ref_port.py): every truncation, every framing-bit flip, value-bit flips, length-prefix edits,
packed-varint terminators and same-length framing edits of every seed.  The walker must refuse exactly what the runtime
refuses - except a malformed packed varint, which is opaque to the walk and reported by the varint decode kernels - and
otherwise tabulate what the runtime parses, output for output.  This pins the reference the GPU tests compare against.
"""
import numpy as np
import pytest
from google.protobuf.message import DecodeError

import decode_mutants as D
from min_tfs_client import _native as N
from min_tfs_client.constants import numpy_for_enum
from oracle import ref_port
from tensorflow.core.framework import tensor_pb2
from tensorflow_serving.apis import predict_pb2

SEEDS = D.seeds()
_STATUS_OF = {ValueError: N.E_SHAPE, KeyError: N.E_KEY}


def _reference(tp):
    """tensor_proto_to_ndarray on one parsed TensorProto: the array, or the class of the exception it raises."""
    try:
        return ref_port.from_tensor_proto(tp)
    except (ValueError, KeyError, TypeError) as e:
        return type(e)


def _check_output(m, w, k, tp, what):
    o = w.outs[k]
    assert o.dtype == tp.dtype, what
    assert w.dims[k] == [d.size for d in tp.tensor_shape.dim], what
    ref = _reference(tp)
    if isinstance(ref, type):
        if ref is TypeError:             # rank 0: reshape() without arguments, whatever the values; the walker flags it
            assert o.flags & N.OF_RANK0 and o.rank == 0, what
        elif ref is UnicodeDecodeError:
            assert o.dtype == 7 and o.status == N.OK, what      # string values are unpacked on the host, which raises the same
        elif ref is KeyError and o.dtype == 14:
            assert o.status in (N.OK, N.E_SHAPE), what        # DT_BFLOAT16: tabulated; the strict decode raises KeyError for it
        elif ref is ValueError and o.status == N.OK and o.flags & N.OF_VARINT:
            # packed varints: the walk checks the element count only as far as value bytes allow; the varint decode kernels
            # count the terminators and report the mismatch when the output is unpacked
            raw = D.run_bytes(m.buf, w.runs[k])
            assert sum(1 for b in raw if not b & 0x80) != o.n_elems, what
        else:
            assert o.status == _STATUS_OF[ref], (what, o.status, ref)
        return
    if o.status == N.OK and (o.flags & N.OF_VARINT) and ref.size == 0:
        return
    assert o.status == N.OK, (what, o.status)
    assert numpy_for_enum(o.dtype) == ref.dtype.type, what
    if o.dtype in D.FIXED:
        assert D.fixed_values(m.buf, w, k) == ref.tobytes(), what
    elif o.flags & N.OF_VARINT:
        raw = D.run_bytes(m.buf, w.runs[k])
        assert sum(1 for b in raw if not b & 0x80) == ref.size, what      # one terminator per element
    else:
        assert o.n_strings == ref.size, what


def _check_spec(rec, spec, ms):
    def text(off, n):
        return rec[off: off + n].decode()
    assert text(spec.name_off, spec.name_len) == ms.name
    assert text(spec.signature_off, spec.signature_len) == ms.signature_name
    assert bool(spec.has_version) == ms.HasField("version") and (not spec.has_version or spec.version == ms.version.value)
    assert text(spec.label_off, spec.label_len) == ms.version_label


def check_mutant(m):
    """The walker against the protobuf runtime + ref_port for one mutant; returns the walker's record status."""
    rec = m.record
    w = D.walk(m.buf, m.rec_len, tensor=m.tensor)
    what = (m.seed, m.kind, m.rec_len)
    try:
        parsed = (tensor_pb2.TensorProto if m.tensor else predict_pb2.PredictResponse).FromString(rec)
    except DecodeError:
        # Either the walk refuses the record, or a packed-varint payload is malformed INSIDE (value bytes are opaque to the
        # walk): the varint decode kernels report that when the output is unpacked
        assert w.status == N.E_PARSE or (w.status == N.OK and any(D.malformed_varints(m.buf, w, k) for k in range(len(w.outs)))), \
            (what, w.status)
        return w.status
    assert w.status == N.OK, ("the runtime accepts these bytes but the walker rejected them", what, w.status)
    if m.tensor:
        _check_output(m, w, 0, parsed, what)
        return w.status
    keys = [rec[o.key_off: o.key_off + o.key_len].decode() for o in w.outs]
    assert sorted(keys) == sorted(parsed.outputs), what
    for k, key in enumerate(keys):
        _check_output(m, w, k, parsed.outputs[key], what + (key,))
    _check_spec(rec, w.spec, parsed.model_spec)
    return w.status


@pytest.mark.parametrize("seed", SEEDS, ids=[s.name for s in SEEDS])
def test_walker_agrees_with_the_runtime_on_every_mutant(seed):
    ms = D.mutants(seed)
    kinds = {}
    for m in ms:
        st = check_mutant(m)
        ok, total = kinds.get(m.kind, (0, 0))
        kinds[m.kind] = (ok + (st == N.OK), total + 1)
    print(seed.name, len(ms), "mutants;", ", ".join(f"{k} {ok}/{t} ok" for k, (ok, t) in sorted(kinds.items())))
    # each seed must exercise what it is there for: refused and accepted records, and the walks the template must not cover
    assert any(st_ok < tot for st_ok, tot in kinds.values()) and any(st_ok for st_ok, _ in kinds.values())


def test_same_length_edits_parse_to_another_table_and_miss_the_template():
    """Every same-length framing edit is a valid record with another table; the template restatement refuses it, while
    accepting every value-byte flip that keeps packed varints terminated."""
    n_edits = 0
    for s in SEEDS:
        if s.tensor:
            continue
        t = D.template_of(s.wire)
        base = D.walk(s.wire, len(s.wire))
        for label, e in s.edits:
            w = D.walk(e, len(e))
            assert w.status == N.OK, (s.name, label)
            def keys(rec, walk):
                return [rec[o.key_off: o.key_off + o.key_len] for o in walk.outs]
            differs = len(w.outs) != len(base.outs) or w.dims != base.dims or w.runs != base.runs or any(
                bytes(a) != bytes(b) for a, b in zip(w.outs, base.outs)) or keys(e, w) != keys(s.wire, base) or \
                D.spec_text(e, w.spec) != D.spec_text(s.wire, base.spec)
            assert differs, (s.name, label)
            if t is not None:
                assert not D.verdict(t, e, len(e)), (s.name, label)
            n_edits += 1
        if t is not None:
            for m in D.mutants(s):
                if m.kind == "value_flip":
                    w = D.walk(m.buf, m.rec_len, max_outputs=N.FUSED_MAX_OUTPUTS, spill=False)
                    if D.verdict(t, m.buf, m.rec_len):
                        assert w.status == N.OK and [bytes(o) for o in w.outs] == [bytes(o) for o in D.walk(s.wire, len(s.wire), max_outputs=8, spill=False).outs]
    assert n_edits >= 25


def test_corpus_covers_the_device_only_code():
    """Seeds longer than two cache lines with framing in three or more of them, records ending on both sides of a line
    boundary, seeds large enough for several 32 KB tiles, and templates for every response seed but the spilling one."""
    lines, tiles, ends = [], [], set()
    for s in SEEDS:
        w = D.walk(s.wire, len(s.wire), tensor=s.tensor)
        value = np.zeros(len(s.wire), dtype=bool)
        for a, b in D.value_ranges(w):
            value[a:b] = True
        if len({int(i) >> 7 for i in np.flatnonzero(~value)}) >= 3:
            lines.append(s.name)
        if len(s.wire) >= 2 * 32768:
            tiles.append(s.name)
        ends.add(len(s.wire) % 128)
        if not s.tensor and s.name != "spill":
            assert D.template_of(s.wire) is not None, s.name
    assert "evict" in lines and len(tiles) >= 3 and {127, 0, 1} <= ends, (lines, tiles, ends)


@D.EXHAUSTIVE
def test_every_value_flip_of_the_large_seeds(request):
    D.require_exhaustive(request.config)
    for s in SEEDS:
        if len(s.wire) > D.SMALL:
            for m in D.value_flips(s):
                check_mutant(m)
