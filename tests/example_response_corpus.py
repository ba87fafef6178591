"""Classify / Regress responses for the example-response decode tests: what a server writes, the edge cases the runtime's
behaviour pins, and a seeded mutant corpus around them.  Shared by the host-walk test (CPU) and the device decode test (GPU).

Responses are built as trees of ``(field, wire_type, payload)`` nodes - payload: bytes for scalars and strings, a list of nodes
for a sub-message; ``(None, RAW, bytes)`` is emitted verbatim - so that a mutant can lie about one particular length or spell
one particular varint in more bytes than it needs.
"""
import random
import struct

import numpy as np

REGRESS, CLASSIFY = 1, 2          # B200TFS_RESP_*
VARINT, I64, LEN, SGROUP, EGROUP, I32 = 0, 1, 2, 3, 4, 5
RAW = "raw"


def varint(v: int, pad: int = 0) -> bytes:
    """v as a varint; `pad` extra bytes make it non-minimal (still the same value)."""
    out = []
    while True:
        b, v = v & 0x7F, v >> 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            break
    if pad:
        out[-1] |= 0x80
        out += [0x80] * (pad - 1) + [0x00]
    return bytes(out)


def f32(x) -> bytes:
    return struct.pack("<f", x) if isinstance(x, float) else struct.pack("<I", x)


def serialize(nodes, mut=None, ctr=None) -> bytes:
    """mut: None, ("len", k, delta) - the k-th length says delta more -, ("pad_len", k) or ("pad_tag", k)."""
    ctr = {"tag": 0, "len": 0} if ctr is None else ctr
    out = bytearray()
    for f, wt, p in nodes:
        if wt == RAW:
            out += p
            continue
        t = ctr["tag"]
        ctr["tag"] += 1
        out += varint(f << 3 | wt, 1 if mut == ("pad_tag", t) else 0)
        if wt == LEN:
            body = serialize(p, mut, ctr) if isinstance(p, list) else p
            k = ctr["len"]
            ctr["len"] += 1
            n = len(body)
            if mut and mut[0] == "len" and mut[1] == k and n + mut[2] >= 0:
                n += mut[2]
            out += varint(n, 1 if mut == ("pad_len", k) else 0) + body
        else:
            out += p
    return bytes(out)


def count(nodes, what) -> int:
    ctr = {"tag": 0, "len": 0}
    serialize(nodes, None, ctr)
    return ctr[what]


def spec_nodes(name=b"model", version=None, signature=b"", label=None):
    s = [(1, LEN, name)]
    if version is not None:
        s.append((2, LEN, [(1, VARINT, varint(version & (2 ** 64 - 1)))]))
    if label is not None:
        s.append((4, LEN, label))
    if signature:
        s.append((3, LEN, signature))
    return [(2, LEN, s)]


def regression_nodes(values, spec=True, spec_first=False):
    """A RegressionResponse as a server writes it: +0.0 elided (an empty Regression), anything else as `0D f32`."""
    regs = [(1, LEN, [] if struct.pack("<f", v) == b"\0\0\0\0" else [(1, I32, f32(v))]) for v in values]
    body = [(1, LEN, regs)]
    sp = spec_nodes(version=3, signature=b"serving_default") if spec else []
    return sp + body if spec_first else body + sp


def classification_nodes(examples, spec=True):
    """examples: a list of [(label bytes, score)] per example."""
    cls = []
    for ex in examples:
        classes = []
        for label, score in ex:
            c = []
            if label:
                c.append((1, LEN, label))
            if struct.pack("<f", score) != b"\0\0\0\0":
                c.append((2, I32, f32(score)))
            classes.append((1, LEN, c))
        cls.append((1, LEN, classes))
    return [(1, LEN, cls)] + (spec_nodes(version=1, signature=b"serving_default") if spec else [])


# ---- the runtime's behaviour, case by case ---------------------------------------------------------------------------------
def edge_cases():
    """(name, kind, wire): every case the decode must match FromString on."""
    G = [(9, SGROUP, b""), (None, RAW, bytes([1 << 3 | 0, 1, 2 << 3 | 5, 1, 2, 3, 4])), (9, EGROUP, b"")]
    unknown = [(15, VARINT, varint(300)), (16, I64, b"\1" * 8), (17, I32, b"\2" * 4), (18, LEN, b"zz")] + G
    cases = [
        ("regress_empty", REGRESS, b""),
        ("regress_no_result", REGRESS, serialize(spec_nodes())),
        ("regress_empty_result", REGRESS, serialize([(1, LEN, [])])),
        ("regress_zero_elided", REGRESS, serialize(regression_nodes([0.0, 1.5]))),
        ("regress_neg_zero", REGRESS, serialize(regression_nodes([-0.0]))),
        ("regress_snan", REGRESS, serialize([(1, LEN, [(1, LEN, [(1, I32, f32(0x7F800001))])])])),
        ("regress_spec_first", REGRESS, serialize(regression_nodes([1.0, 2.0], spec_first=True))),
        ("regress_dup_value", REGRESS, serialize([(1, LEN, [(1, LEN, [(1, I32, f32(1.0)), (1, I32, f32(2.0))])])])),
        ("regress_wrong_wire_type", REGRESS, serialize([(1, LEN, [(1, LEN, [(1, VARINT, varint(5))])])])),
        ("regress_unknown_everywhere", REGRESS, serialize(unknown + [(1, LEN, unknown + [(1, LEN, unknown + [(1, I32, f32(4.0))] + unknown)])]
                                                          + spec_nodes() + unknown)),
        ("regress_repeated_result", REGRESS, serialize(regression_nodes([1.0, 2.0]) + [(1, LEN, [(1, LEN, [(1, I32, f32(3.0))])])])),
        ("regress_repeated_spec", REGRESS, serialize(regression_nodes([1.0]) + spec_nodes(name=b"other", label=b"canary"))),
        ("regress_result_wrong_wire_type", REGRESS, serialize([(1, VARINT, varint(7))] + regression_nodes([1.0]))),
        ("classify_empty", CLASSIFY, b""),
        ("classify_no_classes", CLASSIFY, serialize(classification_nodes([[], []]))),
        ("classify_empty_class", CLASSIFY, serialize([(1, LEN, [(1, LEN, [(1, LEN, [])])])])),
        ("classify_basic", CLASSIFY, serialize(classification_nodes([[(b"a", 0.25), (b"b", 0.75)], [(b"a", -0.0), (b"b", 0.0)]]))),
        ("classify_utf8", CLASSIFY, serialize(classification_nodes([[("ß".encode(), 1.0), ("€".encode(), 2.0), ("😀".encode(), 3.0), (b"", 4.0)]]))),
        ("classify_dup_label_score", CLASSIFY, serialize([(1, LEN, [(1, LEN, [(1, LEN, [(1, LEN, b"x"), (2, I32, f32(1.0)), (1, LEN, b"y"),
                                                                                   (2, I32, f32(2.0))])])])])),
        ("classify_label_emptied", CLASSIFY, serialize([(1, LEN, [(1, LEN, [(1, LEN, [(1, LEN, b"x"), (1, LEN, b"")])])])])),
        ("classify_wrong_wire_types", CLASSIFY, serialize([(1, LEN, [(1, LEN, [(1, LEN, [(1, I32, f32(1.0)), (2, VARINT, varint(3))]),
                                                                            (1, VARINT, varint(1))])])])),
        ("classify_unknown_everywhere", CLASSIFY, serialize(unknown + [(1, LEN, unknown + [(1, LEN, unknown + [(1, LEN, unknown + [(1, LEN, b"q")]
                                                                                                                     + unknown)])])])),
        ("classify_repeated_result", CLASSIFY, serialize(classification_nodes([[(b"a", 1.0)]]) + [(1, LEN, [(1, LEN, [(1, LEN, [(1, LEN, b"b")])])])])),
        ("classify_ragged", CLASSIFY, serialize(classification_nodes([[(b"a", 1.0), (b"b", 2.0)], [(b"a", 1.0)]]))),
        ("classify_bad_utf8", CLASSIFY, serialize(classification_nodes([[(b"\xff", 1.0)]]))),
        ("classify_overlong_utf8", CLASSIFY, serialize(classification_nodes([[(b"\xc0\x80", 1.0)]]))),
        ("classify_surrogate", CLASSIFY, serialize(classification_nodes([[(b"\xed\xa0\x80", 1.0)]]))),
        ("classify_past_max", CLASSIFY, serialize(classification_nodes([[(b"\xf4\x90\x80\x80", 1.0)]]))),
        ("classify_cut_utf8", CLASSIFY, serialize(classification_nodes([[(b"\xe2\x82", 1.0)]]))),
        ("spec_bad_utf8", REGRESS, serialize(regression_nodes([1.0], spec=False) + spec_nodes(name=b"\xff"))),
        ("tag_zero", REGRESS, b"\x00\x00"),
        ("wire_type_6", REGRESS, b"\x0e"),
        ("wire_type_7", CLASSIFY, b"\x0f"),
        ("stray_end_group", REGRESS, b"\x0c"),
        ("mismatched_group", REGRESS, bytes([9 << 3 | 3, 10 << 3 | 4])),
        ("open_group", REGRESS, bytes([9 << 3 | 3])),
        ("varint_11_bytes", REGRESS, bytes([15 << 3]) + b"\xff" * 10 + b"\x01"),
        ("varint_10_bytes", REGRESS, bytes([15 << 3]) + b"\xff" * 9 + b"\x01"),
        ("length_past_end", REGRESS, b"\x0a\x05\x0a\x00"),
        ("truncated_value", REGRESS, b"\x0a\x04\x0a\x02\x0d\x00"),
    ]
    return cases + long_tag_cases()


def long_tag(field: int, wt: int, n: int) -> bytes:
    """the tag of (field, wt) written in n bytes (n at least its minimal length)"""
    t = varint(field << 3 | wt)
    return varint(field << 3 | wt, n - len(t)) if n > len(t) else t


def tag_5th_byte(field: int, wt: int, top: int) -> bytes:
    """a 5-byte tag of (field, wt) whose last byte is `top`: bits 28 and up of the value (0x0F: it still fits 32 bits, 0x10: it
    does not)"""
    v = field << 3 | wt
    return bytes([(v & 0x7F) | 0x80, (v >> 7 & 0x7F) | 0x80, (v >> 14 & 0x7F) | 0x80, (v >> 21 & 0x7F) | 0x80, top])


def long_tag_cases():
    """(name, kind, wire): tags written in 2 to 10 bytes at every level the decode reads one.  The runtime accepts a tag of at
    most 5 bytes whose value fits 32 bits, and refuses every longer one, whatever its value."""
    v = f32(1.5)
    cases = []
    for n in range(2, 11):
        e = long_tag(1, LEN, n)
        cases += [
            (f"result_tag_{n}_bytes", REGRESS, e + b"\x07" + b"\x0a\x05\x0d" + v),
            (f"entry_tag_{n}_bytes", REGRESS, serialize([(1, LEN, [(None, RAW, e + b"\x05\x0d" + v), (1, LEN, [(1, I32, v)])])])),
            (f"value_tag_{n}_bytes", REGRESS, serialize([(1, LEN, [(1, LEN, [(None, RAW, long_tag(1, I32, n) + v)])])])),
            (f"unknown_tag_{n}_bytes", REGRESS, long_tag(15, VARINT, n) + b"\x01" + serialize(regression_nodes([2.0]))),
            (f"unknown_body_tag_{n}_bytes", REGRESS, serialize([(1, LEN, [(None, RAW, long_tag(15, I64, n) + b"\1" * 8), (1, LEN, [])])])),
            (f"group_member_tag_{n}_bytes", REGRESS, serialize([(1, LEN, [(9, SGROUP, b""), (None, RAW, long_tag(1, VARINT, n) + b"\x01"),
                                                                          (9, EGROUP, b""), (1, LEN, [])])])),
            (f"class_tag_{n}_bytes", CLASSIFY, serialize([(1, LEN, [(1, LEN, [(None, RAW, e + b"\x03\x0a\x01a"),
                                                                              (1, LEN, [(1, LEN, b"b")])])])])),
            (f"label_tag_{n}_bytes", CLASSIFY, serialize([(1, LEN, [(1, LEN, [(1, LEN, [(None, RAW, e + b"\x01a")])])])])),
        ]
    for top in (0x0F, 0x10):
        t = tag_5th_byte(1, LEN, top)            # field (1 | 0x0F << 25) or a value past 32 bits: never an entry
        cases += [
            (f"unknown_tag_5th_byte_{top:02x}", REGRESS, t + b"\x00" + serialize(regression_nodes([3.0]))),
            (f"unknown_body_tag_5th_byte_{top:02x}", REGRESS, serialize([(1, LEN, [(None, RAW, t + b"\x01z"), (1, LEN, [(1, I32, v)])])])),
            (f"unknown_class_tag_5th_byte_{top:02x}", CLASSIFY, serialize([(1, LEN, [(1, LEN, [(1, LEN, [(None, RAW, t + b"\x00"),
                                                                                                         (1, LEN, b"a")])])])])),
        ]
    return cases


def _bases():
    rng = random.Random(7)
    vals = [1.5, -0.0, 0.0, float("inf"), 0x7F800001, 3.25]
    reg = regression_nodes([v if isinstance(v, float) else struct.unpack("<f", f32(v))[0] for v in vals])
    reg_raw = [(1, LEN, [(1, LEN, [(1, I32, f32(v))]) for v in (1.0, 0x7FA00000, 2.0)])] + spec_nodes(name=b"r", version=-2, signature=b"s")
    cls = classification_nodes([[(b"cat", 0.5), ("dög".encode(), -1.0)], [(b"cat", 0.25), (b"", 2.0)]])
    extra = [(15, VARINT, varint(rng.randrange(1 << 20))), (9, SGROUP, b""), (None, RAW, b"\x08\x01"), (9, EGROUP, b"")]
    cls_unknown = [(1, LEN, [(1, LEN, [(1, LEN, [(1, LEN, b"x"), (2, I32, f32(1.0))] + extra)] + extra)] + extra)] + spec_nodes()
    return [(REGRESS, reg), (REGRESS, reg_raw), (CLASSIFY, cls), (CLASSIFY, cls_unknown)]


def mutants():
    """(kind, wire) pairs: every truncation, every bit flip of every byte, every length +-1 and +-128, every tag and length
    spelled non-minimally, unknown fields and duplicates inserted, wrong wire types, invalid UTF-8 labels - around the bases."""
    out = []
    for kind, nodes in _bases():
        w = serialize(nodes)
        out += [(kind, w[:i]) for i in range(len(w))]
        for i in range(len(w)):
            for b in range(8):
                m = bytearray(w)
                m[i] ^= 1 << b
                out.append((kind, bytes(m)))
        for k in range(count(nodes, "len")):
            out += [(kind, serialize(nodes, ("len", k, d))) for d in (-128, -1, 1, 128)]
            out.append((kind, serialize(nodes, ("pad_len", k))))
        out += [(kind, serialize(nodes, ("pad_tag", k))) for k in range(count(nodes, "tag"))]
        out.append((kind, w + w))                                      # everything twice: results and specs merge
        out.append((kind, w + bytes([20 << 3 | 3, 21 << 3 | 3, 21 << 3 | 4, 20 << 3 | 4])))
        out.append((kind, w + bytes([1 << 3 | 0, 1])))                 # result with the wrong wire type
    for bad in (b"\xff", b"\xc3", b"\xe0\x80\x80", b"\xed\xbf\xbf", b"\xf8\x88\x80\x80\x80", b"a\x80"):
        out.append((CLASSIFY, serialize(classification_nodes([[(b"ok", 1.0), (bad, 2.0)]]))))
    return out


def random_regression(rng: np.random.Generator, n: int) -> bytes:
    from tensorflow_serving.apis.regression_pb2 import RegressionResponse

    r = RegressionResponse()
    r.model_spec.name = "m"
    r.result.SetInParent()
    for v in rng.standard_normal(n).astype(np.float32):
        r.result.regressions.add(value=float(v))
    return r.SerializeToString()


def random_classification(rng: np.random.Generator, n: int, labels) -> bytes:
    """n examples; labels: a list of C labels (every example) or a callable (example index -> labels)."""
    from tensorflow_serving.apis.classification_pb2 import ClassificationResponse

    r = ClassificationResponse()
    r.model_spec.name = "m"
    r.result.SetInParent()
    for i in range(n):
        cl = r.result.classifications.add()
        ls = labels(i) if callable(labels) else labels
        for lab, s in zip(ls, rng.standard_normal(len(ls)).astype(np.float32)):
            cl.classes.add(label=lab, score=float(s))
    return r.SerializeToString()


def expected(kind: int, wires):
    """The definition: (values / scores, labels, counts) from FromString, or the DecodeError / ValueError it leads to."""
    from tensorflow_serving.apis.classification_pb2 import ClassificationResponse
    from tensorflow_serving.apis.regression_pb2 import RegressionResponse

    if kind == REGRESS:
        ms = [RegressionResponse.FromString(w) for w in wires]
        vals = np.array([r.value for m in ms for r in m.result.regressions], np.float32)
        return vals, None, [len(m.result.regressions) for m in ms]
    ms = [ClassificationResponse.FromString(w) for w in wires]
    rows = [[(c.label, c.score) for c in cl.classes] for m in ms for cl in m.result.classifications]
    if len({len(r) for r in rows}) > 1:
        raise ValueError("examples disagree on the number of classes")
    C = len(rows[0]) if rows else 0
    scores = np.array([[s for _, s in r] for r in rows], np.float32).reshape(len(rows), C)
    return scores, [[lab for lab, _ in r] for r in rows], [len(m.result.classifications) for m in ms]
