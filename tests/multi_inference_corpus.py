"""MultiInference responses for the MultiInference decode tests: what a server writes, the edge cases the runtime's behaviour pins,
a seeded mutant corpus around them, and the definition every decode is held against.  Shared by the host-walk test (CPU) and
the device decode test (GPU).  Built with example_response_corpus's node serializer: an InferenceResult is
``[(1, LEN, model_spec)] + [(2 | 3, LEN, ClassificationResult | RegressionResult body)]``."""
import numpy as np

import example_response_corpus as X
from example_response_corpus import EGROUP, I32, I64, LEN, RAW, SGROUP, VARINT, f32, serialize, varint

REGRESS, CLASSIFY = X.REGRESS, X.CLASSIFY
CLS, REG = 2, 3                    # InferenceResult's oneof members


def spec(name=b"model", version=None, signature=b"", label=None):
    """an InferenceResult's model_spec field (1)"""
    return [(1, LEN, X.spec_nodes(name, version, signature, label)[0][2])]


def cls_body(examples):
    return X.classification_nodes(examples, spec=False)[0][2]


def reg_body(values):
    return X.regression_nodes(values, spec=False)[0][2]


def result(member=None, body=None, sp=True, sig=b"serving_default"):
    """one `results` field: the model_spec, then the member's body"""
    nodes = spec(version=1, signature=sig) if sp else []
    if member is not None:
        nodes = nodes + [(member, LEN, body)]
    return (1, LEN, nodes)


EX2 = [[(b"pos", 0.25), (b"neg", 0.75)], [(b"pos", -0.0), (b"neg", 0.0)]]
UNKNOWN = [(15, VARINT, varint(300)), (16, I64, b"\1" * 8), (17, I32, b"\2" * 4), (18, LEN, b"zz"), (9, SGROUP, b""),
           (None, RAW, bytes([1 << 3 | 0, 1, 2 << 3 | 5, 1, 2, 3, 4])), (9, EGROUP, b"")]


def edge_cases():
    """(name, kinds, wire): every case the decode must match the definition on."""
    C, R = CLASSIFY, REGRESS
    cr = [result(CLS, cls_body(EX2)), result(REG, reg_body([1.5, -0.0, 2.0]))]
    return [
        ("plain", [C, R], serialize(cr)),
        ("one_task", [R], serialize([result(REG, reg_body([3.0]))])),
        ("oneof_2_3", [R], serialize([(1, LEN, spec() + [(CLS, LEN, cls_body(EX2)), (REG, LEN, reg_body([4.0]))])])),
        ("oneof_3_2", [C], serialize([(1, LEN, spec() + [(REG, LEN, reg_body([4.0])), (CLS, LEN, cls_body(EX2))])])),
        ("oneof_2_3_2", [C], serialize([(1, LEN, [(CLS, LEN, cls_body([[(b"a", 1.0)]])), (REG, LEN, reg_body([4.0])),
                                                   (CLS, LEN, cls_body([[(b"b", 2.0)]]))])])),
        ("oneof_2_3_2_as_regress", [R], serialize([(1, LEN, [(CLS, LEN, cls_body([[(b"a", 1.0)]])), (REG, LEN, reg_body([4.0])),
                                                             (CLS, LEN, cls_body([[(b"b", 2.0)]]))])])),
        ("member_merge", [R, C], serialize([(1, LEN, [(REG, LEN, reg_body([1.0])), (REG, LEN, reg_body([2.0, 3.0]))]),
                                            (1, LEN, [(CLS, LEN, cls_body([[(b"a", 1.0)]])), (20, VARINT, varint(1)),
                                                      (CLS, LEN, cls_body([[(b"a", 5.0)]]))])])),
        ("spec_merge", [R], serialize([(1, LEN, spec(name=b"m", version=7) + [(REG, LEN, reg_body([1.0]))]
                                        + spec(name=b"", signature=b"sig", label=b"lab"))])),
        ("unknown_everywhere", [C, R], serialize(UNKNOWN + [(1, LEN, UNKNOWN + spec() + [(CLS, LEN, UNKNOWN + cls_body(EX2) + UNKNOWN)]
                                                              + UNKNOWN)] + UNKNOWN
                                                 + [(1, LEN, [(REG, LEN, reg_body([1.0]) + UNKNOWN)] + UNKNOWN)] + UNKNOWN)),
        ("member_wrong_wire_type", [R], serialize([(1, LEN, [(CLS, VARINT, varint(1)), (REG, LEN, reg_body([1.0])), (CLS, I32, f32(1.0))])])),
        ("results_wrong_wire_type", [R], serialize([(1, VARINT, varint(3)), result(REG, reg_body([1.0]))])),
        ("zero_results", [R], b""),
        ("zero_results_two_tasks", [C, R], serialize(UNKNOWN)),
        ("fewer_results", [C, R], serialize(cr[:1])),
        ("more_results", [C], serialize(cr)),
        ("wrong_case", [R, C], serialize(cr)),
        ("empty_result", [R], serialize([(1, LEN, [])])),
        ("empty_result_spec_only", [C], serialize([result(sp=True)])),
        ("empty_bodies", [C, R], serialize([result(CLS, []), result(REG, [])])),
        ("ragged_classes", [C], serialize([result(CLS, cls_body([[(b"a", 1.0), (b"b", 2.0)], [(b"a", 1.0)]]))])),
        ("cleared_bad_utf8", [R], serialize([(1, LEN, [(CLS, LEN, cls_body([[(b"\xff", 1.0)]])), (REG, LEN, reg_body([1.0]))])])),
        ("cleared_truncated_value", [C], serialize([(1, LEN, [(REG, LEN, [(1, LEN, [(1, I32, b"\0\0")])]), (CLS, LEN, cls_body(EX2))])])),
        ("past_tasks_bad_utf8", [R], serialize([result(REG, reg_body([1.0])), result(CLS, cls_body([[(b"\xc0\x80", 1.0)]]))])),
        ("wrong_case_bad_utf8", [R], serialize([result(CLS, cls_body([[(b"\xed\xa0\x80", 1.0)]]))])),
        ("decoded_bad_utf8", [C], serialize([result(CLS, cls_body([[(b"ok", 1.0)], [(b"\xff", 2.0)]]))])),
        ("spec_bad_utf8", [R], serialize([(1, LEN, spec(name=b"\xff") + [(REG, LEN, reg_body([1.0]))])])),
        ("snan", [R, C], serialize([result(REG, [(1, LEN, [(1, I32, f32(0x7F800001))])]),
                                    result(CLS, [(1, LEN, [(1, LEN, [(1, LEN, b"x"), (2, I32, f32(0xFFA00000))])])])])),
        ("tag_zero", [R], b"\x00\x00"),
        ("length_past_end", [R], b"\x0a\x05\x1a\x00"),
        ("open_group", [R], serialize([result(REG, reg_body([1.0]))]) + bytes([9 << 3 | 3])),
    ]


def _bases():
    vals = [1.5, -0.0, 0.0, float("inf"), 3.25]
    a = [result(CLS, cls_body([[(b"cat", 0.5), ("dög".encode(), -1.0)], [(b"cat", 0.25), (b"", 2.0)]])), result(REG, reg_body(vals))]
    extra = [(15, VARINT, varint(77)), (9, SGROUP, b""), (None, RAW, b"\x08\x01"), (9, EGROUP, b"")]
    b = [(1, LEN, spec(name=b"r", version=-2, signature=b"s") + [(REG, LEN, reg_body([9.0])), (CLS, LEN, cls_body([[(b"x", 1.0)]]) + extra),
                                                                   (CLS, LEN, cls_body([[(b"y", 2.0)]]))] + extra),
         (1, LEN, [(REG, LEN, [(1, LEN, [(1, I32, f32(v))]) for v in (1.0, 0x7FA00000)] + extra)])]
    return [([CLASSIFY, REGRESS], a), ([CLASSIFY, REGRESS], b)]


def mutants():
    """(kinds, wire): every truncation, every bit flip, every length +-1 and +-128, non-minimal tags and lengths, everything twice,
    around the bases."""
    out = []
    for kinds, nodes in _bases():
        w = serialize(nodes)
        out += [(kinds, w[:i]) for i in range(len(w))]
        for i in range(len(w)):
            for bit in range(8):
                m = bytearray(w)
                m[i] ^= 1 << bit
                out.append((kinds, bytes(m)))
        for k in range(X.count(nodes, "len")):
            out += [(kinds, serialize(nodes, ("len", k, d))) for d in (-128, -1, 1, 128)]
            out.append((kinds, serialize(nodes, ("pad_len", k))))
        out += [(kinds, serialize(nodes, ("pad_tag", k))) for k in range(X.count(nodes, "tag"))]
        out.append((kinds, w + w))
        out.append((kinds[:1], w))
    return out


def random_response(rng: np.random.Generator, kinds, n: int, labels=("pos", "neg"), name="m") -> bytes:
    """What a server writes: one result per task, in task order, each with the model_spec and n examples."""
    from tensorflow_serving.apis.inference_pb2 import MultiInferenceResponse

    r = MultiInferenceResponse()
    for t, k in enumerate(kinds):
        res = r.results.add()
        res.model_spec.name = name
        res.model_spec.version.value = 3
        res.model_spec.signature_name = f"head{t}"
        if k == REGRESS:
            res.regression_result.SetInParent()
            for v in rng.standard_normal(n).astype(np.float32):
                res.regression_result.regressions.add(value=float(v))
        else:
            res.classification_result.SetInParent()
            for i in range(n):
                cl = res.classification_result.classifications.add()
                ls = labels(i) if callable(labels) else labels
                for lab, s in zip(ls, rng.standard_normal(len(ls)).astype(np.float32)):
                    cl.classes.add(label=lab, score=float(s))
    return r.SerializeToString()


def expected(kinds, wires):
    """The definition: per task (values / scores, labels or None, counts, model_specs), or the DecodeError / ValueError it raises."""
    from tensorflow_serving.apis.inference_pb2 import MultiInferenceResponse

    msgs = [MultiInferenceResponse.FromString(bytes(w)) for w in wires]
    T = len(kinds)
    for m in msgs:
        if len(m.results) != T:
            raise ValueError("result count")
        for t, k in enumerate(kinds):
            if m.results[t].WhichOneof("result") != ("classification_result" if k == CLASSIFY else "regression_result"):
                raise ValueError("result case")
    out = []
    for t, k in enumerate(kinds):
        specs = [m.results[t].model_spec for m in msgs]
        if k == REGRESS:
            res = [m.results[t].regression_result for m in msgs]
            out.append((np.array([g.value for r in res for g in r.regressions], np.float32), None, [len(r.regressions) for r in res], specs))
            continue
        res = [m.results[t].classification_result for m in msgs]
        rows = [[(c.label, c.score) for c in cl.classes] for r in res for cl in r.classifications]
        if len({len(r) for r in rows}) > 1:
            raise ValueError("examples disagree on the number of classes")
        nc = len(rows[0]) if rows else 0
        scores = np.array([[s for _, s in r] for r in rows], np.float32).reshape(len(rows), nc)
        out.append((scores, [[lab for lab, _ in r] for r in rows], [len(r.classifications) for r in res], specs))
    return out
