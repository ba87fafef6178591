"""Reference bytes of a PredictRequest whose one input is a DT_STRING vector of serialized tf.Examples, built with the protobuf
runtime: model_spec as ``_make_inference_request`` sets it, ``inputs[key]`` = DT_STRING of shape [n] whose ``string_val`` holds
``e.SerializeToString(deterministic=True)`` of every example ``examples_from_input_dict`` builds (one example at a time, as
ragged_ref does, when a column is ragged), the request serialized with ``deterministic=True``."""
from min_tfs_client.codec import RaggedColumn
from min_tfs_client.requests import examples_from_input_dict
from ragged_ref import host
from tensorflow.core.framework import types_pb2
from tensorflow_serving.apis.predict_pb2 import PredictRequest


def examples(d):
    """the tf.Examples of input_dict d (numpy or torch columns, RaggedColumn included)"""
    cols = {k: (host(v.values), host(v.lengths)) if isinstance(v, RaggedColumn) else host(v) for k, v in d.items()}
    if not any(isinstance(v, tuple) for v in cols.values()):
        return list(examples_from_input_dict(cols).example_list.examples)
    n = {v[0].shape[0] if isinstance(v, tuple) else v.shape[0] for v in cols.values() if isinstance(v, tuple) or v.ndim}.pop()
    out = []
    for i in range(n):
        one = {k: v[0][i:i + 1, :int(v[1][i])] if isinstance(v, tuple) else v if v.ndim == 0 else v[i:i + 1] for k, v in cols.items()}
        out += examples_from_input_dict(one).example_list.examples
    return out


def predict_examples_request(name, version, d, key="examples") -> PredictRequest:
    req = PredictRequest()
    req.model_spec.name = name
    if version is not None:
        req.model_spec.version.value = version
    ex = examples(d)
    t = req.inputs[key.decode("utf-8") if isinstance(key, bytes) else key]
    t.dtype = types_pb2.DT_STRING
    t.tensor_shape.dim.add().size = len(ex)
    t.string_val.extend(e.SerializeToString(deterministic=True) for e in ex)
    return req


def predict_examples_ref(name, version, d, key="examples", grpc_frame=False) -> bytes:
    wire = predict_examples_request(name, version, d, key).SerializeToString(deterministic=True)
    return (b"\x00" + len(wire).to_bytes(4, "big") + wire) if grpc_frame else wire
