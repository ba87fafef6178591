"""Drop-in for the Predict part of the reference's ``min_tfs_client/requests.py``.

``TensorServingClient(host, port, credentials=None).predict_request(model_name, input_dict,
timeout=60, model_version=None)`` keeps the reference's signature (requests.py:22-65).  The request
is packed by the encode kernels and sent as raw bytes through the same gRPC method the generated stub
binds (``/tensorflow.serving.PredictionService/Predict``, prediction_service_pb2_grpc.py:50-54); the
response bytes are handed to the parse/unpack kernels.

The reference's other three calls are kept as well (requests.py:67-110).  They are outside the Predict hot path
(SURVEY.md 8(f) rank 4): small pointer-chasing messages assembled on the host by the protobuf runtime, like
``DT_STRING`` tensors.  ``model_status_request`` is the reference's; ``classification_request`` /
``regression_request`` cannot work in the reference (it fills ``request.inputs[k]``, a field neither
``ClassificationRequest`` nor ``RegressionRequest`` has, and sends them to ``Predict``): here they build the
``Input{example_list}`` those RPCs define - one ``tf.Example`` per row of ``input_dict`` - and call
``PredictionService/Classify`` and ``/Regress``.
"""
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .codec import BytesColumn, RaggedColumn, _sequence_count, get_codec
from .tensors import WireTensor

PREDICT_METHOD = "/tensorflow.serving.PredictionService/Predict"
CLASSIFY_METHOD = "/tensorflow.serving.PredictionService/Classify"
REGRESS_METHOD = "/tensorflow.serving.PredictionService/Regress"
MULTI_INFERENCE_METHOD = "/tensorflow.serving.PredictionService/MultiInference"
MODEL_STATUS_METHOD = "/tensorflow.serving.ModelService/GetModelStatus"
# the method names of a MultiInference task (TF's signature_constants CLASSIFY_METHOD_NAME / REGRESS_METHOD_NAME)
CLASSIFY_METHOD_NAME = "tensorflow/serving/classify"
REGRESS_METHOD_NAME = "tensorflow/serving/regress"


def examples_from_input_dict(input_dict: Dict[str, np.ndarray]):
    """``Input{example_list{examples}}`` for Classify / Regress (input.proto:13-79, example.proto, feature.proto).

    Row i of every array is example i: ``feature[k]`` holds the row's values flattened - ``float_list`` for floating
    dtypes, ``int64_list`` for integers and bools, ``bytes_list`` for str / bytes (``coerce_to_bytes``).  0-d arrays are
    repeated in every example; all other arrays must agree on their first dimension.  A ``RaggedColumn`` gives example i
    only ``values[i, :lengths[i]]``.  A ``BytesColumn`` (or a ``RaggedColumn`` of one) gives example i its strings, as they are.
    """
    from tensorflow_serving.apis.input_pb2 import Input

    arrays = {k: v if isinstance(v, (RaggedColumn, BytesColumn)) else np.asarray(v) for k, v in input_dict.items()}
    rows = {a.shape[0] for a in arrays.values() if a.ndim}
    if len(rows) > 1:
        raise ValueError(f"inputs disagree on the number of examples: {sorted(rows)}")
    n = rows.pop() if rows else (1 if arrays else 0)
    inp = Input()
    inp.example_list.SetInParent()
    for i in range(n):
        _fill_example(inp.example_list.examples.add(), arrays, i)
    return inp


def _fill_example(ex, arrays: Dict, i: int) -> None:
    """Example ``ex`` holds row i of every array (0-d arrays: their one value), as ``examples_from_input_dict`` fills it."""
    for k, a in arrays.items():
        feat = ex.features.feature[k]
        if isinstance(a, BytesColumn) or isinstance(a, RaggedColumn) and isinstance(a.values, BytesColumn):
            feat.bytes_list.value.extend(a.strings(i))
            continue
        _fill_feature(feat, k, a.row(i) if isinstance(a, RaggedColumn) else a if a.ndim == 0 else a[i])


def _fill_feature(feat, k, row: np.ndarray) -> None:
    """``feat`` holds ``row`` flattened in C order: ``float_list`` for floating dtypes, ``int64_list`` for integers and bools,
    ``bytes_list`` for str / bytes."""
    from .tensors import coerce_to_bytes

    if row.dtype.kind == "f":
        feat.float_list.value.extend(np.asarray(row, dtype=np.float32).ravel().tolist())
    elif row.dtype.kind in "iub":
        feat.int64_list.value.extend(np.asarray(row, dtype=np.int64).ravel().tolist())
    elif row.dtype.kind in "US":
        feat.bytes_list.value.extend(coerce_to_bytes(s) for s in np.asarray(row).ravel().tolist())
    else:
        raise ValueError(f"input {k!r}: dtype {row.dtype} has no tf.Example feature kind")


def examples_with_context_from_input_dict(input_dict: Dict[str, np.ndarray], context_dict: Dict[str, np.ndarray]):
    """``Input{example_list_with_context{examples, context}}`` (input.proto ExampleListWithContext): what a ranking or
    recommendation model takes for Classify / Regress - the candidates' examples, as ``examples_from_input_dict`` builds them, and
    one context Example shared by all of them.  Context feature ``k`` holds the whole of ``context_dict[k]`` flattened in C order
    (a 0-d array is one value), converted as an example's values are; a ``BytesColumn`` gives all its strings.  An empty
    ``context_dict`` is an empty context, which is still sent.  A ``RaggedColumn`` raises ValueError: a context has no example
    axis."""
    from tensorflow_serving.apis.input_pb2 import Input

    inp = Input()
    elwc = inp.example_list_with_context
    elwc.examples.extend(examples_from_input_dict(input_dict).example_list.examples)
    elwc.context.SetInParent()
    for k, v in context_dict.items():
        if isinstance(v, RaggedColumn):
            raise ValueError(f"context {k!r}: a RaggedColumn has no place in a context, which has no example axis")
        feat = elwc.context.features.feature[k]
        if isinstance(v, BytesColumn):
            o = np.asarray(v.offsets).tolist()
            d = np.asarray(v.data)
            feat.bytes_list.value.extend(d[o[j]: o[j + 1]].tobytes() for j in range(len(o) - 1))
        else:
            _fill_feature(feat, k, np.asarray(v))
    return inp


def _list_steps(a, i: int) -> list:
    """The steps of sequence i of a feature-list value of shape ``[n, T, *inner]`` (a ``RaggedColumn``: its first ``lengths[i]``):
    arrays of shape ``inner``, or for a ``BytesColumn`` lists of the step's strings."""
    vals = a.values if isinstance(a, RaggedColumn) else a
    steps = int(a.lengths[i]) if isinstance(a, RaggedColumn) else a.shape[1]
    if isinstance(vals, BytesColumn):
        unit = int(np.prod(vals.shape[2:], dtype=np.int64))
        strs = vals.strings(i, steps * unit)
        return [strs[t * unit:(t + 1) * unit] for t in range(steps)]
    row = np.asarray(vals)[i]
    return [row[t] for t in range(steps)]


def sequence_examples_from_input_dict(context_dict: Dict[str, np.ndarray], feature_list_dict: Dict[str, np.ndarray]) -> list:
    """One ``tf.SequenceExample`` per sequence (example.proto, feature.proto FeatureLists): what a model exported with a
    ``tf.io.parse_sequence_example`` serving input takes.  Context feature ``k`` of sequence i is filled as
    ``examples_from_input_dict`` fills example i's (row i; a 0-d value repeated in every sequence; ``RaggedColumn`` and
    ``BytesColumn`` values as there).  A feature-list value has shape ``[n, T, *inner]`` (an array, a ``BytesColumn``, or a
    ``RaggedColumn`` of either, whose sequence i has ``lengths[i]`` steps): sequence i's ``feature_list[f]`` holds one Feature per
    step, step t holding ``value[i, t]`` flattened (a bytes value: the step's strings).  A list of no steps still has its entry, and
    ``context`` and ``feature_lists`` are always set.  n is the leading dimension every non-0-d context value and every feature-list
    value share (ValueError when they disagree, or for a feature-list value of rank < 2); with none, 1 when a dict is non-empty."""
    from tensorflow.core.example.example_pb2 import SequenceExample

    n = _sequence_count(context_dict, feature_list_dict)
    ctx = {k: v if isinstance(v, (RaggedColumn, BytesColumn)) else np.asarray(v) for k, v in context_dict.items()}
    lists = {k: v if isinstance(v, (RaggedColumn, BytesColumn)) else np.asarray(v) for k, v in feature_list_dict.items()}
    out = []
    for i in range(n):
        s = SequenceExample()
        s.context.SetInParent()
        s.feature_lists.SetInParent()
        for k, a in ctx.items():
            feat = s.context.feature[k]
            if isinstance(a, BytesColumn) or isinstance(a, RaggedColumn) and isinstance(a.values, BytesColumn):
                feat.bytes_list.value.extend(a.strings(i))
                continue
            _fill_feature(feat, k, a.row(i) if isinstance(a, RaggedColumn) else a if a.ndim == 0 else a[i])
        for k, a in lists.items():
            fl = s.feature_lists.feature_list[k]
            for step in _list_steps(a, i):
                if isinstance(step, list):
                    fl.feature.add().bytes_list.value.extend(step)
                else:
                    _fill_feature(fl.feature.add(), k, step)
        out.append(s)
    return out


def _list_sizes(list_sizes) -> np.ndarray:
    """The host int64 vector of a batch's list sizes (ValueError when it is not a 1-D integer array, or has a negative size)."""
    sizes = np.asarray(list_sizes)
    if sizes.ndim != 1 or (sizes.size and sizes.dtype.kind not in "iu"):
        raise ValueError(f"list_sizes is a 1-D integer array, got {sizes.dtype} of shape {sizes.shape}")
    sizes = np.ascontiguousarray(sizes, dtype=np.int64)
    if (sizes < 0).any():
        raise ValueError("list sizes must be >= 0")
    return sizes


def elwcs_from_input_dict(context_dict, input_dict, list_sizes) -> list:
    """One ``ExampleListWithContext`` per query (input.proto): what TF-Ranking's ELWC serving signature takes as a DT_STRING
    ``[None]`` vector, one serialized ELWC per query.  ``list_sizes`` is a 1-D integer array of Q sizes >= 0 (Q may be 0), and n
    their sum.  Example j (j < n) holds row j of every non-0-d value of ``input_dict``, filled as ``examples_from_input_dict``
    fills it (0-d values repeated; ``RaggedColumn`` and ``BytesColumn`` values as there); query q's examples are the
    ``list_sizes[q]`` rows from ``sum(list_sizes[:q])`` on.  Context q holds row q of every non-0-d value of ``context_dict``
    the same way (0-d values repeated, ``RaggedColumn`` and ``BytesColumn`` values allowed), and is always set: an empty
    ``context_dict`` gives empty contexts.  ValueError when an input value's leading dim is not n, a context value's is not Q,
    or a list size is negative."""
    from tensorflow_serving.apis.input_pb2 import ExampleListWithContext

    sizes = _list_sizes(list_sizes)
    n = int(sizes.sum())

    def rows(d, m, what):
        arrays = {k: v if isinstance(v, (RaggedColumn, BytesColumn)) else np.asarray(v) for k, v in d.items()}
        for k, a in arrays.items():
            if a.ndim and a.shape[0] != m:
                raise ValueError(f"{what} {k!r} has {a.shape[0]} rows, not {m}")
        return arrays

    inputs, ctx = rows(input_dict, n, "input"), rows(context_dict, sizes.size, "context")
    out, s = [], 0
    for q, m in enumerate(sizes.tolist()):
        e = ExampleListWithContext()
        for j in range(s, s + m):
            _fill_example(e.examples.add(), inputs, j)
        e.context.SetInParent()
        _fill_example(e.context, ctx, q)
        out.append(e)
        s += m
    return out


def make_predict_elwcs_request(model_name: str, model_version: Optional[int], context_dict, input_dict, list_sizes, input_key: str, *,
                               signature_name=None, version_label=None, output_filter=None):
    """``PredictRequest`` whose one input ``input_key`` is the DT_STRING ``[Q]`` tensor of the ExampleListWithContexts
    ``elwcs_from_input_dict`` builds, each serialized with ``deterministic=True`` - several TF-Ranking queries in one Predict
    call, what ``Codec.encode_elwc_requests`` encodes on the GPU.  ``signature_name``, ``version_label`` and ``output_filter``
    set those fields (``apply_spec_fields``)."""
    from tensorflow.core.framework.types_pb2 import DT_STRING
    from tensorflow_serving.apis.predict_pb2 import PredictRequest

    req = PredictRequest()
    req.model_spec.name = model_name
    if model_version is not None:
        req.model_spec.version.value = model_version
    elwcs = elwcs_from_input_dict(context_dict, input_dict, list_sizes)
    t = req.inputs[input_key.decode("utf-8") if isinstance(input_key, bytes) else input_key]
    t.dtype = DT_STRING
    t.tensor_shape.dim.add().size = len(elwcs)
    t.string_val.extend(e.SerializeToString(deterministic=True) for e in elwcs)
    return apply_spec_fields(req, model_version, signature_name, version_label, output_filter)


class SpecFields(dict):
    """``signature_name`` / ``version_label`` / ``output_filter`` as the last element of a ``gpu_*_serializer`` request tuple."""


def _split_fields(request):
    """(the request tuple without its SpecFields, the fields as keywords)"""
    if request and isinstance(request[-1], SpecFields):
        return tuple(request[:-1]), dict(request[-1])
    return tuple(request), {}


def _fields(signature_name=None, version_label=None, output_filter=None) -> SpecFields:
    return SpecFields({k: v for k, v in dict(signature_name=signature_name, version_label=version_label,
                                             output_filter=output_filter).items() if v is not None})


def apply_spec_fields(req, model_version=None, signature_name=None, version_label=None, output_filter=None):
    """Set ``signature_name``, ``version_label`` and ``output_filter`` (None: left unset) on a request protobuf builds: every
    task's model_spec of a MultiInferenceRequest (whose tasks carry their own signatures), else the request's model_spec.
    ValueError, as ``Codec`` raises it, for a label beside a version, bytes that are not UTF-8, a filter on a request that is not
    a PredictRequest and a signature beside tasks."""
    from .codec import _RequestSpec

    s = _RequestSpec.of([model_version], signature_name, version_label, output_filter)
    if s is None:
        return req
    sig, label, names = s.keep[0], s.keep[1], s.keep[2]
    multi = req.DESCRIPTOR.name == "MultiInferenceRequest"
    if multi and signature_name is not None:
        raise ValueError("a MultiInference request names a signature per task, not one for the whole request")
    if output_filter is not None and req.DESCRIPTOR.name != "PredictRequest":
        raise ValueError("output_filter is a PredictRequest field: a Classify, Regress or MultiInference request has none")
    for spec in [t.model_spec for t in req.tasks] if multi else [req.model_spec]:
        if sig:
            spec.signature_name = sig.decode("utf-8")
        if label is not None:
            spec.version_label = label.decode("utf-8")
    if output_filter is not None:
        req.output_filter.extend(x.decode("utf-8") for x in names)
    return req


def make_predict_sequence_examples_request(model_name: str, model_version: Optional[int], context_dict, feature_list_dict,
                                           input_key: str, *, signature_name=None, version_label=None, output_filter=None):
    """``PredictRequest`` whose one input ``input_key`` is the DT_STRING ``[n]`` tensor of the sequences
    ``sequence_examples_from_input_dict`` builds, each serialized with ``deterministic=True`` - what
    ``Codec.encode_sequence_example_requests`` encodes on the GPU.  ``signature_name``, ``version_label`` and ``output_filter``
    set those fields (``apply_spec_fields``)."""
    from tensorflow.core.framework.types_pb2 import DT_STRING
    from tensorflow_serving.apis.predict_pb2 import PredictRequest

    req = PredictRequest()
    req.model_spec.name = model_name
    if model_version is not None:
        req.model_spec.version.value = model_version
    seqs = sequence_examples_from_input_dict(context_dict, feature_list_dict)
    t = req.inputs[input_key.decode("utf-8") if isinstance(input_key, bytes) else input_key]
    t.dtype = DT_STRING
    t.tensor_shape.dim.add().size = len(seqs)
    t.string_val.extend(s.SerializeToString(deterministic=True) for s in seqs)
    return apply_spec_fields(req, model_version, signature_name, version_label, output_filter)


def _checked_tasks(tasks) -> List[Tuple[str, str]]:
    """The MultiInference tasks ``[(signature_name, method_name), ...]`` with None signatures as "" and bytes ones decoded;
    ValueError for no task or a method name other than CLASSIFY_METHOD_NAME / REGRESS_METHOD_NAME."""
    out = []
    for sig, method in tasks:
        if method not in (CLASSIFY_METHOD_NAME, REGRESS_METHOD_NAME):
            raise ValueError(f"task method {method!r} is neither {CLASSIFY_METHOD_NAME!r} nor {REGRESS_METHOD_NAME!r}")
        out.append(("" if sig is None else sig.decode("utf-8") if isinstance(sig, bytes) else str(sig), method))
    if not out:
        raise ValueError("a MultiInferenceRequest needs at least one task")
    return out


def make_multi_inference_request(model_name: str, model_version: Optional[int], tasks: Sequence[Tuple[str, str]],
                                 input_dict: Dict[str, np.ndarray], context_dict=None, *, signature_name=None, version_label=None,
                                 output_filter=None):
    """``MultiInferenceRequest`` (inference.proto) running every task ``(signature_name, method_name)`` of the model over one
    Input: ``examples_from_input_dict(input_dict)``, or with ``context_dict`` ``examples_with_context_from_input_dict``.  Each
    task's model_spec names the model, the version (when not None) and the signature (an empty or None one: not set, the server's
    default); its method_name is ``CLASSIFY_METHOD_NAME`` or ``REGRESS_METHOD_NAME`` (anything else raises ValueError, as does an
    empty task list).  What ``Codec.encode_example_requests(..., tasks=...)`` encodes on the GPU.  ``version_label`` goes into every
    task's model_spec behind its signature; ``signature_name`` (each task names its own) and ``output_filter`` (a PredictRequest
    field) raise ValueError."""
    from tensorflow_serving.apis.inference_pb2 import MultiInferenceRequest

    req = MultiInferenceRequest()
    for sig, method in _checked_tasks(tasks):
        t = req.tasks.add()
        t.model_spec.SetInParent()
        t.model_spec.name = model_name
        if model_version is not None:
            t.model_spec.version.value = model_version
        if sig:
            t.model_spec.signature_name = sig
        t.method_name = method
    if context_dict is None:
        req.input.CopyFrom(examples_from_input_dict(input_dict))
    else:
        req.input.CopyFrom(examples_with_context_from_input_dict(input_dict, context_dict))
    return apply_spec_fields(req, model_version, signature_name, version_label, output_filter)


class PredictResponseView:
    """What ``predict_request`` returns: ``.outputs[key]`` (decode with ``tensor_proto_to_ndarray``),
    ``.model_spec``; anything else is answered by a real ``PredictResponse`` parsed on demand."""

    def __init__(self, wire: bytes):
        self._wire = wire
        self._proto = None
        self._views = None

    def to_proto(self):
        if self._proto is None:
            from tensorflow_serving.apis.predict_pb2 import PredictResponse

            self._proto = PredictResponse.FromString(self._wire)
        return self._proto

    @property
    def outputs(self) -> Dict[str, WireTensor]:
        if self._views is None:
            opened = get_codec().open_predict_response(self._wire)   # one launch decodes every fixed-width output
            if opened is not None:
                self._views = {k: WireTensor(opened=opened, key=k) for k in opened.table}
            else:   # empty / malformed / more outputs than the fused launch tabulates: the two-phase path (raises like FromString)
                parsed = get_codec().parse_predict_responses([self._wire])[0]
                buf, base = parsed.wire, parsed.offset
                self._views = {k: WireTensor(buf[base + o.msg_off: base + o.msg_off + o.msg_len].tobytes()) for k, o in parsed.outputs.items()}
        return self._views

    def to_ndarrays(self, **options) -> Dict[str, np.ndarray]:
        """Every output decoded in one parse + one unpack launch."""
        return get_codec().decode_predict_response(self._wire, **options)[0]

    def SerializeToString(self) -> bytes:  # noqa: N802
        return self._wire

    def __getattr__(self, name):
        return getattr(self.to_proto(), name)


class _ExampleResponseView:
    """A Classify / Regress response decoded on the GPU on first use; anything the view does not answer itself comes from a
    real response message parsed on demand."""

    _message = None      # the protobuf class

    def __init__(self, wire: bytes):
        self._wire = wire
        self._proto = None
        self._batch = None

    def to_proto(self):
        if self._proto is None:
            self._proto = self._message.FromString(self._wire)
        return self._proto

    def SerializeToString(self) -> bytes:  # noqa: N802
        return self._wire

    def __getattr__(self, name):
        return getattr(self.to_proto(), name)


class ClassificationResponseView(_ExampleResponseView):
    """What ``gpu_classification_response_deserializer`` returns: ``.scores`` (float32 ``[examples, classes]``) and
    ``.labels()`` decoded by the kernels; ``.result``, ``.model_spec``, ... from a ``ClassificationResponse``."""

    from tensorflow_serving.apis.classification_pb2 import ClassificationResponse as _message

    def _decoded(self):
        if self._batch is None:
            self._batch = get_codec().decode_classification_responses([self._wire])
        return self._batch

    @property
    def scores(self) -> np.ndarray:
        return self._decoded().scores

    def labels(self):
        return self._decoded().labels()


class RegressionResponseView(_ExampleResponseView):
    """What ``gpu_regression_response_deserializer`` returns: ``.values`` (float32 ``[examples]``) decoded by the kernels;
    ``.result``, ``.model_spec``, ... from a ``RegressionResponse``."""

    from tensorflow_serving.apis.regression_pb2 import RegressionResponse as _message

    @property
    def values(self) -> np.ndarray:
        if self._batch is None:
            self._batch = get_codec().decode_regression_responses([self._wire])
        return self._batch.values


def gpu_classification_response_deserializer(wire: bytes) -> ClassificationResponseView:
    """``response_deserializer`` for ``channel.unary_unary(CLASSIFY_METHOD, ...)``: bytes -> lazy response view."""
    return ClassificationResponseView(wire)


def gpu_regression_response_deserializer(wire: bytes) -> RegressionResponseView:
    """``response_deserializer`` for ``channel.unary_unary(REGRESS_METHOD, ...)``: bytes -> lazy response view."""
    return RegressionResponseView(wire)


def gpu_request_serializer(request) -> bytes:
    """``request_serializer`` for ``channel.unary_unary``: (model_name, model_version, input_dict[, spec]) -> bytes.  A DT_STRING input
    may be a numpy str array (UTF-8, as the reference) or a ``BytesColumn`` of host arrays, whose strings go out as their raw bytes -
    how a request carries binary data such as encoded images.  ``spec``, a dict of ``signature_name`` / ``version_label`` /
    ``output_filter``, sets those fields (``Codec.encode_predict_requests``)."""
    request, spec = _split_fields(request)
    model_name, model_version, input_dict = request[:3]
    spec.update(request[3] if len(request) > 3 else {})
    return get_codec().encode_predict_request(model_name, input_dict, model_version, **spec)


def gpu_example_request_serializer(request) -> bytes:
    """``request_serializer`` for ``channel.unary_unary(CLASSIFY_METHOD | REGRESS_METHOD, ...)``: (model_name, model_version,
    input_dict[, context_dict]) -> the ClassificationRequest / RegressionRequest bytes ``_make_example_request`` would serialise,
    packed on the GPU (with a context_dict that is not None: an ExampleListWithContext).  A trailing ``SpecFields`` sets
    ``signature_name`` / ``version_label``."""
    request, spec = _split_fields(request)
    return get_codec().encode_example_requests([request], **spec)[0]


def gpu_predict_examples_serializer(request) -> bytes:
    """``request_serializer`` for ``channel.unary_unary(PREDICT_METHOD, ...)`` to a model that parses serialized tf.Examples:
    (model_name, model_version, input_dict, input_key) -> a PredictRequest whose input ``input_key`` is the DT_STRING ``[n]``
    tensor of the examples ``examples_from_input_dict`` builds, each serialized with ``deterministic=True``, packed on the GPU.
    (..., input_key, context_dict) with a context_dict that is not None: the input is instead the DT_STRING ``[1]`` tensor of the
    one ExampleListWithContext ``examples_with_context_from_input_dict`` builds (TF-Ranking's serving input)."""
    request, spec = _split_fields(request)
    model_name, model_version, input_dict, input_key = request[:4]
    context_dict = request[4] if len(request) > 4 else None
    return get_codec().encode_example_requests([(model_name, model_version, input_dict, context_dict)], predict_input=input_key,
                                               **spec)[0]


def gpu_multi_inference_request_serializer(request) -> bytes:
    """``request_serializer`` for ``channel.unary_unary(MULTI_INFERENCE_METHOD, ...)``: (model_name, model_version, tasks,
    input_dict[, context_dict]) -> the bytes of ``make_multi_inference_request(...).SerializeToString(deterministic=True)``,
    packed on the GPU."""
    request, spec = _split_fields(request)
    model_name, model_version, tasks, input_dict = request[:4]
    context_dict = request[4] if len(request) > 4 else None
    return get_codec().encode_example_requests([(model_name, model_version, input_dict, context_dict)], tasks=tasks, **spec)[0]


def gpu_predict_sequence_examples_serializer(request) -> bytes:
    """``request_serializer`` for ``channel.unary_unary(PREDICT_METHOD, ...)`` to a model that parses serialized
    tf.SequenceExamples: (model_name, model_version, context_dict, feature_list_dict, input_key) -> the bytes of
    ``make_predict_sequence_examples_request(...).SerializeToString(deterministic=True)``, packed on the GPU."""
    request, spec = _split_fields(request)
    model_name, model_version, context_dict, feature_list_dict, input_key = request
    return get_codec().encode_sequence_example_requests([(model_name, model_version, context_dict, feature_list_dict)],
                                                        input_key=input_key, **spec)[0]


def gpu_predict_elwcs_serializer(request) -> bytes:
    """``request_serializer`` for ``channel.unary_unary(PREDICT_METHOD, ...)`` to a TF-Ranking model's ELWC signature:
    (model_name, model_version, context_dict, input_dict, list_sizes, input_key) -> the bytes of
    ``make_predict_elwcs_request(...).SerializeToString(deterministic=True)``, packed on the GPU.  ``list_sizes`` may be a device
    int64 vector over a capacity of input rows (``Codec.encode_elwc_requests``).  A trailing ``SpecFields`` sets
    ``signature_name`` / ``version_label`` / ``output_filter``."""
    request, spec = _split_fields(request)
    model_name, model_version, context_dict, input_dict, list_sizes, input_key = request
    return get_codec().encode_elwc_requests([(model_name, model_version, context_dict, input_dict, list_sizes)], input_key=input_key,
                                            **spec)[0]


def gpu_response_deserializer(wire: bytes) -> PredictResponseView:
    """``response_deserializer`` for ``channel.unary_unary``: bytes -> lazy response view."""
    return PredictResponseView(wire)


# grpc's default receive limit is 4 MiB and the reference leaves it alone (requests.py:27-30): a response that carries a
# fp32[1024,1024] tensor (4 194 3xx bytes) is refused with RESOURCE_EXHAUSTED.  Pass these to lift both limits.
LARGE_MESSAGE_CHANNEL_OPTIONS = (("grpc.max_send_message_length", -1), ("grpc.max_receive_message_length", -1))


class TensorServingClient:
    def __init__(self, host: str, port: int, credentials=None, channel_options=None) -> None:
        """Same arguments as the reference (requests.py:22-30); ``channel_options`` (default None: grpc's defaults, like the
        reference) is handed to ``grpc.insecure_channel`` / ``grpc.secure_channel``, e.g. ``LARGE_MESSAGE_CHANNEL_OPTIONS``."""
        import grpc

        self._host_address = f"{host}:{port}"
        options = list(channel_options) if channel_options else None
        if credentials:
            self._channel = grpc.secure_channel(self._host_address, credentials, options=options)
        else:
            self._channel = grpc.insecure_channel(self._host_address, options=options)
        self._predict = self._channel.unary_unary(PREDICT_METHOD, request_serializer=gpu_request_serializer,
                                                  response_deserializer=gpu_response_deserializer)

    def predict_request(self, model_name: str, input_dict: Dict[str, np.ndarray], timeout: int = 60,
                        model_version: Optional[int] = None, *, signature_name=None, version_label=None,
                        output_filter=None) -> PredictResponseView:
        """The reference's signature (requests.py:32-65), plus ``signature_name`` (a signature other than the server's default),
        ``version_label`` (a labelled version such as ``"canary"``; not with ``model_version``) and ``output_filter`` (only these
        outputs are computed and returned)."""
        return self._predict((model_name, model_version, input_dict, _fields(signature_name, version_label, output_filter)), timeout)

    def predict_examples_request(self, model_name: str, input_dict: Dict[str, np.ndarray], input_key: str = "examples",
                                 timeout: int = 60, model_version: Optional[int] = None, context_dict=None, *, signature_name=None,
                                 version_label=None, output_filter=None) -> PredictResponseView:
        """Predict on a model whose signature takes serialized tf.Examples (a DT_STRING vector it parses with
        ``tf.io.parse_example``, e.g. a TFX Trainer or Estimator export's ``serving_default``): one example per row of
        ``input_dict`` as ``examples_from_input_dict`` builds it, sent as input ``input_key``.  Values may be ``RaggedColumn`` and
        ``BytesColumn`` columns, encoded on the GPU like the numeric ones.  With ``context_dict`` the input is one serialized
        ExampleListWithContext instead (a TF-Ranking model's serving input), the context holding the whole of each value."""
        call = self._channel.unary_unary(PREDICT_METHOD, request_serializer=gpu_predict_examples_serializer,
                                         response_deserializer=gpu_response_deserializer)
        return call((model_name, model_version, input_dict, input_key, context_dict, _fields(signature_name, version_label, output_filter)),
                    timeout)

    def predict_sequence_examples_request(self, model_name: str, context_dict, feature_list_dict, input_key: str, timeout: int = 60,
                                          model_version: Optional[int] = None, *, signature_name=None, version_label=None,
                                          output_filter=None) -> PredictResponseView:
        """Predict on a model whose signature takes serialized tf.SequenceExamples (a DT_STRING vector it parses with
        ``tf.io.parse_sequence_example``: a session or event-history model, or TF-Ranking's SequenceExample format): one sequence
        per row, as ``sequence_examples_from_input_dict(context_dict, feature_list_dict)`` builds it, sent as input
        ``input_key`` and packed on the GPU."""
        call = self._channel.unary_unary(PREDICT_METHOD, request_serializer=gpu_predict_sequence_examples_serializer,
                                         response_deserializer=gpu_response_deserializer)
        return call((model_name, model_version, context_dict, feature_list_dict, input_key,
                     _fields(signature_name, version_label, output_filter)), timeout)

    def predict_elwcs_request(self, model_name: str, context_dict, input_dict, list_sizes, input_key: str, timeout: int = 60,
                              model_version: Optional[int] = None, *, signature_name=None, version_label=None,
                              output_filter=None) -> PredictResponseView:
        """Predict on a TF-Ranking model whose signature takes a DT_STRING vector of serialized ExampleListWithContexts, one per
        query: the Q = ``len(list_sizes)`` ELWCs ``elwcs_from_input_dict(context_dict, input_dict, list_sizes)`` builds, sent as
        input ``input_key`` in one call and packed on the GPU.  ``list_sizes`` may be a device int64 vector, as a GPU candidate
        stage leaves it: the rows of ``input_dict`` are then a capacity, and the rows past the sizes' total are not sent
        (``Codec.encode_elwc_requests``)."""
        call = self._channel.unary_unary(PREDICT_METHOD, request_serializer=gpu_predict_elwcs_serializer,
                                         response_deserializer=gpu_response_deserializer)
        return call((model_name, model_version, context_dict, input_dict, list_sizes, input_key,
                     _fields(signature_name, version_label, output_filter)), timeout)

    def _make_example_request(self, request_pb, model_name, input_dict, model_version, context_dict=None, signature_name=None,
                              version_label=None):
        request = request_pb()
        request.model_spec.name = model_name
        if model_version is not None:
            request.model_spec.version.value = model_version
        if context_dict is None:
            request.input.CopyFrom(examples_from_input_dict(input_dict))
        else:
            request.input.CopyFrom(examples_with_context_from_input_dict(input_dict, context_dict))
        return apply_spec_fields(request, model_version, signature_name, version_label)

    def classification_request(self, model_name: str, input_dict: Dict[str, np.ndarray], timeout: int = 60,
                               model_version: Optional[int] = None, context_dict=None, *, signature_name=None, version_label=None):
        """Same signature as the reference (requests.py:67-81); returns a ``ClassificationResponse``.  With ``context_dict`` the
        input is an ExampleListWithContext (``examples_with_context_from_input_dict``)."""
        from tensorflow_serving.apis.classification_pb2 import ClassificationRequest, ClassificationResponse

        call = self._channel.unary_unary(CLASSIFY_METHOD, request_serializer=ClassificationRequest.SerializeToString,
                                         response_deserializer=ClassificationResponse.FromString)
        return call(self._make_example_request(ClassificationRequest, model_name, input_dict, model_version, context_dict, signature_name,
                                               version_label), timeout)

    def regression_request(self, model_name: str, input_dict: Dict[str, np.ndarray], timeout: int = 60,
                           model_version: Optional[int] = None, context_dict=None, *, signature_name=None, version_label=None):
        """Same signature as the reference (requests.py:83-97); returns a ``RegressionResponse``.  With ``context_dict`` the
        input is an ExampleListWithContext (``examples_with_context_from_input_dict``)."""
        from tensorflow_serving.apis.regression_pb2 import RegressionRequest, RegressionResponse

        call = self._channel.unary_unary(REGRESS_METHOD, request_serializer=RegressionRequest.SerializeToString,
                                         response_deserializer=RegressionResponse.FromString)
        return call(self._make_example_request(RegressionRequest, model_name, input_dict, model_version, context_dict, signature_name,
                                               version_label), timeout)

    def multi_inference_request(self, model_name: str, input_dict: Dict[str, np.ndarray], tasks: Sequence[Tuple[str, str]],
                                timeout: int = 60, model_version: Optional[int] = None, context_dict=None, *, signature_name=None,
                                version_label=None):
        """``PredictionService/MultiInference``: every task ``(signature_name, method_name)`` of the model - method_name
        ``CLASSIFY_METHOD_NAME`` or ``REGRESS_METHOD_NAME`` - over one Input, one example per row of ``input_dict`` (with
        ``context_dict``: an ExampleListWithContext), the request bytes packed on the GPU.  Returns a ``MultiInferenceResponse``
        (``Codec.decode_multi_inference_responses`` decodes a batch of them on the GPU)."""
        from tensorflow_serving.apis.inference_pb2 import MultiInferenceResponse

        call = self._channel.unary_unary(MULTI_INFERENCE_METHOD, request_serializer=gpu_multi_inference_request_serializer,
                                         response_deserializer=MultiInferenceResponse.FromString)
        return call((model_name, model_version, tasks, input_dict, context_dict, _fields(signature_name, version_label)), timeout)

    def model_status_request(self, model_name: str, model_version: Optional[int] = None, timeout: Optional[int] = 10):
        """``ModelService/GetModelStatus`` as the reference issues it (requests.py:99-110: the version is set only when truthy)."""
        from tensorflow_serving.apis.get_model_status_pb2 import GetModelStatusRequest, GetModelStatusResponse

        request = GetModelStatusRequest()
        request.model_spec.name = model_name
        if model_version:
            request.model_spec.version.value = model_version
        call = self._channel.unary_unary(MODEL_STATUS_METHOD, request_serializer=GetModelStatusRequest.SerializeToString,
                                         response_deserializer=GetModelStatusResponse.FromString)
        return call(request, timeout)
