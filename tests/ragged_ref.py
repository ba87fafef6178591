"""Reference bytes of a Classify / Regress request with ragged columns, built from the unchanged dense code only: example i is
the one example ``examples_from_input_dict`` builds from ``{k: values_k[i:i+1, :lengths_k[i]]}`` for every ragged key,
``{k: x_k[i:i+1]}`` for every dense key and 0-d keys as they are; the examples are merged in order, and the model_spec is
written by ``_make_example_request``."""
import numpy as np

from min_tfs_client.codec import RaggedColumn
from min_tfs_client.requests import TensorServingClient, examples_from_input_dict
from tensorflow_serving.apis.classification_pb2 import ClassificationRequest


def host(v):
    """a host copy of a numpy or torch array"""
    return v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v)


def ragged_ref(name, version, d, grpc_frame=False) -> bytes:
    req = TensorServingClient._make_example_request(None, ClassificationRequest, name, {}, version)
    cols = {k: (host(v.values), host(v.lengths)) if isinstance(v, RaggedColumn) else host(v) for k, v in d.items()}
    n = {v[0].shape[0] if isinstance(v, tuple) else v.shape[0] for v in cols.values() if isinstance(v, tuple) or v.ndim}.pop()
    for i in range(n):
        one = {}
        for k, v in cols.items():
            if isinstance(v, tuple):
                one[k] = v[0][i:i + 1, :int(v[1][i])]
            else:
                one[k] = v if v.ndim == 0 else v[i:i + 1]
        req.input.example_list.examples.extend(examples_from_input_dict(one).example_list.examples)
    wire = req.SerializeToString(deterministic=True)
    return (b"\x00" + len(wire).to_bytes(4, "big") + wire) if grpc_frame else wire
