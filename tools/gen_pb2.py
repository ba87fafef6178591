#!/usr/bin/env python
"""Emit the ``*_pb2.py`` schema modules the drop-in package imports, without ``protoc``.

The reference builds its message classes at install time by running ``protoc`` over the vendored
``.proto`` files (reference ``setup.py:41-49``).  This image has no ``protoc``, so the six files on
the Predict hot path are restated below as a small table, turned into ``FileDescriptorProto``s with
``google.protobuf.descriptor_pb2``, serialised, and written out as ordinary importable modules under
``min-tfs-client_b200/tensorflow{,_serving}/`` - the same module names the reference's generated
code has (``tensorflow.core.framework.tensor_pb2`` ...), so ``min_tfs_client`` imports them the way
the reference does (reference ``tensors.py:2-3``, ``constants.py:5``, ``requests.py:6-14``).

Schema sources restated here (all under reference ``protobuf_srcs/``):
  tensorflow/core/framework/types.proto:12-68            enum DataType
  tensorflow/core/framework/tensor_shape.proto:13-46     TensorShapeProto{Dim}
  tensorflow/core/framework/resource_handle.proto:16-42  ResourceHandleProto
  tensorflow/core/framework/tensor.proto:14-94           TensorProto, VariantTensorDataProto
  tensorflow_serving/apis/model.proto:9-33               ModelSpec
  tensorflow_serving/apis/predict.proto:12-40            PredictRequest / PredictResponse
and, for the client's other RPCs (reference requests.py:67-110), host-side messages only:
  tensorflow/core/example/{feature,example}.proto        tf.Example
  tensorflow_serving/apis/input.proto                    Input{ExampleList}
  tensorflow_serving/apis/{classification,regression}.proto
  tensorflow_serving/apis/inference.proto                MultiInference{Request,Response}
  tensorflow_serving/apis/get_model_status.proto, tensorflow_serving/util/status.proto,
  tensorflow/core/{lib/core,protobuf}/error_codes.proto

``tests/test_schema.py`` checks every field name / number / type / label of the generated modules against a
snapshot of these tables stored in ``tests/golden/schema.json`` (recorded from the generated modules).

Usage:  python tools/gen_pb2.py            (rewrites the modules in place; idempotent)
"""
from __future__ import annotations

import os
import sys

from google.protobuf import descriptor_pb2 as dpb

F = dpb.FieldDescriptorProto
ROOT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "min-tfs-client_b200")

_SCALAR = {
    "int32": F.TYPE_INT32, "int64": F.TYPE_INT64, "uint32": F.TYPE_UINT32, "uint64": F.TYPE_UINT64,
    "float": F.TYPE_FLOAT, "double": F.TYPE_DOUBLE, "bool": F.TYPE_BOOL, "string": F.TYPE_STRING,
    "bytes": F.TYPE_BYTES,
}

# DataType enum: base values, each base value >= 1 also has a `_REF` twin at +100.
_DT_BASE = [
    "INVALID", "FLOAT", "DOUBLE", "INT32", "UINT8", "INT16", "INT8", "STRING", "COMPLEX64", "INT64",
    "BOOL", "QINT8", "QUINT8", "QINT32", "BFLOAT16", "QINT16", "QUINT16", "UINT16", "COMPLEX128",
    "HALF", "RESOURCE", "VARIANT", "UINT32", "UINT64",
]


def _field(msg, name, number, typ, *, repeated=False, packed=None, oneof=None):
    """typ: a scalar keyword, 'enum:<fq name>' or 'msg:<fq name>'."""
    f = msg.field.add(name=name, number=number)
    f.label = F.LABEL_REPEATED if repeated else F.LABEL_OPTIONAL
    if typ in _SCALAR:
        f.type = _SCALAR[typ]
    elif typ.startswith("enum:"):
        f.type, f.type_name = F.TYPE_ENUM, typ[5:]
    elif typ.startswith("msg:"):
        f.type, f.type_name = F.TYPE_MESSAGE, typ[4:]
    else:
        raise ValueError(typ)
    if packed is not None:
        f.options.packed = packed
    if oneof is not None:
        f.oneof_index = oneof
    # json_name as protoc fills it (lowerCamelCase) so descriptors match protoc output
    parts = name.split("_")
    f.json_name = parts[0] + "".join(p[:1].upper() + p[1:] for p in parts[1:])
    return f


def _map_field(msg, name, number, value_type, parent_fq):
    """proto3 `map<string, V> name = number;` = nested <Name>Entry{key=1,value=2} with map_entry."""
    entry_name = "".join(p[:1].upper() + p[1:] for p in name.split("_")) + "Entry"
    entry = msg.nested_type.add(name=entry_name)
    _field(entry, "key", 1, "string")
    _field(entry, "value", 2, value_type)
    entry.options.map_entry = True
    _field(msg, name, number, "msg:%s.%s" % (parent_fq, entry_name), repeated=True)


def build_files():
    files = []

    # ---- types.proto ----------------------------------------------------------------------
    fd = dpb.FileDescriptorProto(name="tensorflow/core/framework/types.proto", package="tensorflow",
                                 syntax="proto3")
    en = fd.enum_type.add(name="DataType")
    for i, base in enumerate(_DT_BASE):
        en.value.add(name="DT_" + base, number=i)
    for i, base in enumerate(_DT_BASE):
        if i:
            en.value.add(name="DT_%s_REF" % base, number=100 + i)
    files.append(fd)

    # ---- tensor_shape.proto ---------------------------------------------------------------
    fd = dpb.FileDescriptorProto(name="tensorflow/core/framework/tensor_shape.proto",
                                 package="tensorflow", syntax="proto3")
    shp = fd.message_type.add(name="TensorShapeProto")
    dim = shp.nested_type.add(name="Dim")
    _field(dim, "size", 1, "int64")
    _field(dim, "name", 2, "string")
    _field(shp, "dim", 2, "msg:.tensorflow.TensorShapeProto.Dim", repeated=True)
    _field(shp, "unknown_rank", 3, "bool")
    files.append(fd)

    # ---- resource_handle.proto ------------------------------------------------------------
    fd = dpb.FileDescriptorProto(name="tensorflow/core/framework/resource_handle.proto",
                                 package="tensorflow", syntax="proto3",
                                 dependency=["tensorflow/core/framework/tensor_shape.proto",
                                             "tensorflow/core/framework/types.proto"])
    rh = fd.message_type.add(name="ResourceHandleProto")
    for n, (nm, ty) in enumerate([("device", "string"), ("container", "string"), ("name", "string"),
                                  ("hash_code", "uint64"), ("maybe_type_name", "string")], start=1):
        _field(rh, nm, n, ty)
    das = rh.nested_type.add(name="DtypeAndShape")
    _field(das, "dtype", 1, "enum:.tensorflow.DataType")
    _field(das, "shape", 2, "msg:.tensorflow.TensorShapeProto")
    _field(rh, "dtypes_and_shapes", 6, "msg:.tensorflow.ResourceHandleProto.DtypeAndShape",
           repeated=True)
    files.append(fd)

    # ---- tensor.proto ---------------------------------------------------------------------
    fd = dpb.FileDescriptorProto(name="tensorflow/core/framework/tensor.proto", package="tensorflow",
                                 syntax="proto3",
                                 dependency=["tensorflow/core/framework/resource_handle.proto",
                                             "tensorflow/core/framework/tensor_shape.proto",
                                             "tensorflow/core/framework/types.proto"])
    tp = fd.message_type.add(name="TensorProto")
    _field(tp, "dtype", 1, "enum:.tensorflow.DataType")
    _field(tp, "tensor_shape", 2, "msg:.tensorflow.TensorShapeProto")
    _field(tp, "version_number", 3, "int32")
    _field(tp, "tensor_content", 4, "bytes")
    # declaration order of the .proto (half_val is declared right after tensor_content)
    _field(tp, "half_val", 13, "int32", repeated=True, packed=True)
    _field(tp, "float_val", 5, "float", repeated=True, packed=True)
    _field(tp, "double_val", 6, "double", repeated=True, packed=True)
    _field(tp, "int_val", 7, "int32", repeated=True, packed=True)
    _field(tp, "string_val", 8, "bytes", repeated=True)
    _field(tp, "scomplex_val", 9, "float", repeated=True, packed=True)
    _field(tp, "int64_val", 10, "int64", repeated=True, packed=True)
    _field(tp, "bool_val", 11, "bool", repeated=True, packed=True)
    _field(tp, "dcomplex_val", 12, "double", repeated=True, packed=True)
    _field(tp, "resource_handle_val", 14, "msg:.tensorflow.ResourceHandleProto", repeated=True)
    _field(tp, "variant_val", 15, "msg:.tensorflow.VariantTensorDataProto", repeated=True)
    _field(tp, "uint32_val", 16, "uint32", repeated=True, packed=True)
    _field(tp, "uint64_val", 17, "uint64", repeated=True, packed=True)
    vt = fd.message_type.add(name="VariantTensorDataProto")
    _field(vt, "type_name", 1, "string")
    _field(vt, "metadata", 2, "bytes")
    _field(vt, "tensors", 3, "msg:.tensorflow.TensorProto", repeated=True)
    files.append(fd)

    # ---- model.proto ----------------------------------------------------------------------
    fd = dpb.FileDescriptorProto(name="tensorflow_serving/apis/model.proto",
                                 package="tensorflow.serving", syntax="proto3",
                                 dependency=["google/protobuf/wrappers.proto"])
    ms = fd.message_type.add(name="ModelSpec")
    ms.oneof_decl.add(name="version_choice")
    _field(ms, "name", 1, "string")
    _field(ms, "version", 2, "msg:.google.protobuf.Int64Value", oneof=0)
    _field(ms, "version_label", 4, "string", oneof=0)
    _field(ms, "signature_name", 3, "string")
    files.append(fd)

    # ---- predict.proto --------------------------------------------------------------------
    fd = dpb.FileDescriptorProto(name="tensorflow_serving/apis/predict.proto",
                                 package="tensorflow.serving", syntax="proto3",
                                 dependency=["tensorflow/core/framework/tensor.proto",
                                             "tensorflow_serving/apis/model.proto"])
    rq = fd.message_type.add(name="PredictRequest")
    _field(rq, "model_spec", 1, "msg:.tensorflow.serving.ModelSpec")
    _map_field(rq, "inputs", 2, "msg:.tensorflow.TensorProto", ".tensorflow.serving.PredictRequest")
    _field(rq, "output_filter", 3, "string", repeated=True)
    rs = fd.message_type.add(name="PredictResponse")
    _field(rs, "model_spec", 2, "msg:.tensorflow.serving.ModelSpec")
    _map_field(rs, "outputs", 1, "msg:.tensorflow.TensorProto", ".tensorflow.serving.PredictResponse")
    files.append(fd)

    # ==== the other RPCs of the reference's client (requests.py:67-110): Classify / Regress / GetModelStatus ====
    # ---- feature.proto / example.proto (tf.Example) ------------------------------------------------
    fd = dpb.FileDescriptorProto(name="tensorflow/core/example/feature.proto", package="tensorflow", syntax="proto3")
    for nm, ty in (("BytesList", "bytes"), ("FloatList", "float"), ("Int64List", "int64")):
        m = fd.message_type.add(name=nm)
        _field(m, "value", 1, ty, repeated=True, packed=None if ty == "bytes" else True)
    ft = fd.message_type.add(name="Feature")
    ft.oneof_decl.add(name="kind")
    _field(ft, "bytes_list", 1, "msg:.tensorflow.BytesList", oneof=0)
    _field(ft, "float_list", 2, "msg:.tensorflow.FloatList", oneof=0)
    _field(ft, "int64_list", 3, "msg:.tensorflow.Int64List", oneof=0)
    fs = fd.message_type.add(name="Features")
    _map_field(fs, "feature", 1, "msg:.tensorflow.Feature", ".tensorflow.Features")
    fl = fd.message_type.add(name="FeatureList")
    _field(fl, "feature", 1, "msg:.tensorflow.Feature", repeated=True)
    fls = fd.message_type.add(name="FeatureLists")
    _map_field(fls, "feature_list", 1, "msg:.tensorflow.FeatureList", ".tensorflow.FeatureLists")
    files.append(fd)

    fd = dpb.FileDescriptorProto(name="tensorflow/core/example/example.proto", package="tensorflow", syntax="proto3",
                                 dependency=["tensorflow/core/example/feature.proto"])
    ex = fd.message_type.add(name="Example")
    _field(ex, "features", 1, "msg:.tensorflow.Features")
    sq = fd.message_type.add(name="SequenceExample")
    _field(sq, "context", 1, "msg:.tensorflow.Features")
    _field(sq, "feature_lists", 2, "msg:.tensorflow.FeatureLists")
    files.append(fd)

    # ---- input.proto ------------------------------------------------------------------------------
    fd = dpb.FileDescriptorProto(name="tensorflow_serving/apis/input.proto", package="tensorflow.serving", syntax="proto3",
                                 dependency=["tensorflow/core/example/example.proto"])
    el = fd.message_type.add(name="ExampleList")
    _field(el, "examples", 1, "msg:.tensorflow.Example", repeated=True)
    ec = fd.message_type.add(name="ExampleListWithContext")
    _field(ec, "examples", 1, "msg:.tensorflow.Example", repeated=True)
    _field(ec, "context", 2, "msg:.tensorflow.Example")
    inp = fd.message_type.add(name="Input")
    inp.oneof_decl.add(name="kind")
    f1 = _field(inp, "example_list", 1, "msg:.tensorflow.serving.ExampleList", oneof=0)
    f1.options.lazy = True
    f2 = _field(inp, "example_list_with_context", 2, "msg:.tensorflow.serving.ExampleListWithContext", oneof=0)
    f2.options.lazy = True
    files.append(fd)

    # ---- classification.proto / regression.proto ---------------------------------------------------
    fd = dpb.FileDescriptorProto(name="tensorflow_serving/apis/classification.proto", package="tensorflow.serving", syntax="proto3",
                                 dependency=["tensorflow_serving/apis/input.proto", "tensorflow_serving/apis/model.proto"])
    cl = fd.message_type.add(name="Class")
    _field(cl, "label", 1, "string")
    _field(cl, "score", 2, "float")
    cs = fd.message_type.add(name="Classifications")
    _field(cs, "classes", 1, "msg:.tensorflow.serving.Class", repeated=True)
    cr = fd.message_type.add(name="ClassificationResult")
    _field(cr, "classifications", 1, "msg:.tensorflow.serving.Classifications", repeated=True)
    rq = fd.message_type.add(name="ClassificationRequest")
    _field(rq, "model_spec", 1, "msg:.tensorflow.serving.ModelSpec")
    _field(rq, "input", 2, "msg:.tensorflow.serving.Input")
    rs = fd.message_type.add(name="ClassificationResponse")
    _field(rs, "model_spec", 2, "msg:.tensorflow.serving.ModelSpec")
    _field(rs, "result", 1, "msg:.tensorflow.serving.ClassificationResult")
    files.append(fd)

    fd = dpb.FileDescriptorProto(name="tensorflow_serving/apis/regression.proto", package="tensorflow.serving", syntax="proto3",
                                 dependency=["tensorflow_serving/apis/input.proto", "tensorflow_serving/apis/model.proto"])
    rg = fd.message_type.add(name="Regression")
    _field(rg, "value", 1, "float")
    rr = fd.message_type.add(name="RegressionResult")
    _field(rr, "regressions", 1, "msg:.tensorflow.serving.Regression", repeated=True)
    rq = fd.message_type.add(name="RegressionRequest")
    _field(rq, "model_spec", 1, "msg:.tensorflow.serving.ModelSpec")
    _field(rq, "input", 2, "msg:.tensorflow.serving.Input")
    rs = fd.message_type.add(name="RegressionResponse")
    _field(rs, "model_spec", 2, "msg:.tensorflow.serving.ModelSpec")
    _field(rs, "result", 1, "msg:.tensorflow.serving.RegressionResult")
    files.append(fd)

    # ---- inference.proto (MultiInference: several Classify / Regress signatures over one Input) -----
    fd = dpb.FileDescriptorProto(name="tensorflow_serving/apis/inference.proto", package="tensorflow.serving", syntax="proto3",
                                 dependency=["tensorflow_serving/apis/classification.proto", "tensorflow_serving/apis/input.proto",
                                             "tensorflow_serving/apis/model.proto", "tensorflow_serving/apis/regression.proto"])
    it = fd.message_type.add(name="InferenceTask")
    _field(it, "model_spec", 1, "msg:.tensorflow.serving.ModelSpec")
    _field(it, "method_name", 2, "string")
    ir = fd.message_type.add(name="InferenceResult")
    ir.oneof_decl.add(name="result")
    _field(ir, "model_spec", 1, "msg:.tensorflow.serving.ModelSpec")
    _field(ir, "classification_result", 2, "msg:.tensorflow.serving.ClassificationResult", oneof=0)
    _field(ir, "regression_result", 3, "msg:.tensorflow.serving.RegressionResult", oneof=0)
    mq = fd.message_type.add(name="MultiInferenceRequest")
    _field(mq, "tasks", 1, "msg:.tensorflow.serving.InferenceTask", repeated=True)
    _field(mq, "input", 2, "msg:.tensorflow.serving.Input")
    ms = fd.message_type.add(name="MultiInferenceResponse")
    _field(ms, "results", 1, "msg:.tensorflow.serving.InferenceResult", repeated=True)
    files.append(fd)

    # ---- error_codes.proto (x2: lib/core re-exports protobuf/) / status.proto / get_model_status.proto ----
    fd = dpb.FileDescriptorProto(name="tensorflow/core/protobuf/error_codes.proto", package="tensorflow.error", syntax="proto3")
    en = fd.enum_type.add(name="Code")
    for nm, num in (("OK", 0), ("CANCELLED", 1), ("UNKNOWN", 2), ("INVALID_ARGUMENT", 3), ("DEADLINE_EXCEEDED", 4), ("NOT_FOUND", 5),
                    ("ALREADY_EXISTS", 6), ("PERMISSION_DENIED", 7), ("UNAUTHENTICATED", 16), ("RESOURCE_EXHAUSTED", 8),
                    ("FAILED_PRECONDITION", 9), ("ABORTED", 10), ("OUT_OF_RANGE", 11), ("UNIMPLEMENTED", 12), ("INTERNAL", 13),
                    ("UNAVAILABLE", 14), ("DATA_LOSS", 15),
                    ("DO_NOT_USE_RESERVED_FOR_FUTURE_EXPANSION_USE_DEFAULT_IN_SWITCH_INSTEAD_", 20)):
        en.value.add(name=nm, number=num)
    files.append(fd)
    fd = dpb.FileDescriptorProto(name="tensorflow/core/lib/core/error_codes.proto", syntax="proto3",
                                 dependency=["tensorflow/core/protobuf/error_codes.proto"])
    fd.public_dependency.append(0)
    files.append(fd)

    fd = dpb.FileDescriptorProto(name="tensorflow_serving/util/status.proto", package="tensorflow.serving", syntax="proto3",
                                 dependency=["tensorflow/core/lib/core/error_codes.proto"])
    sp = fd.message_type.add(name="StatusProto")
    _field(sp, "error_code", 1, "enum:.tensorflow.error.Code").json_name = "error_code"
    _field(sp, "error_message", 2, "string").json_name = "error_message"
    files.append(fd)

    fd = dpb.FileDescriptorProto(name="tensorflow_serving/apis/get_model_status.proto", package="tensorflow.serving", syntax="proto3",
                                 dependency=["tensorflow_serving/apis/model.proto", "tensorflow_serving/util/status.proto"])
    rq = fd.message_type.add(name="GetModelStatusRequest")
    _field(rq, "model_spec", 1, "msg:.tensorflow.serving.ModelSpec")
    mv = fd.message_type.add(name="ModelVersionStatus")
    st = mv.enum_type.add(name="State")
    for nm, num in (("UNKNOWN", 0), ("START", 10), ("LOADING", 20), ("AVAILABLE", 30), ("UNLOADING", 40), ("END", 50)):
        st.value.add(name=nm, number=num)
    _field(mv, "version", 1, "int64")
    _field(mv, "state", 2, "enum:.tensorflow.serving.ModelVersionStatus.State")
    _field(mv, "status", 3, "msg:.tensorflow.serving.StatusProto")
    rs = fd.message_type.add(name="GetModelStatusResponse")
    _field(rs, "model_version_status", 1, "msg:.tensorflow.serving.ModelVersionStatus", repeated=True).json_name = "model_version_status"
    files.append(fd)
    return files


_HEADER = '''# -*- coding: utf-8 -*-
# Schema module written by tools/gen_pb2.py (no protoc in this image).  DO NOT EDIT BY HAND.
# source: {src}
"""Message classes for ``{src}`` built from a serialised FileDescriptorProto."""
from google.protobuf import descriptor_pool as _descriptor_pool
from google.protobuf import symbol_database as _symbol_database
from google.protobuf.internal import builder as _builder
{imports}
_sym_db = _symbol_database.Default()

DESCRIPTOR = _descriptor_pool.Default().AddSerializedFile({blob!r})

_globals = globals()
_builder.BuildMessageAndEnumDescriptors(DESCRIPTOR, _globals)
_builder.BuildTopDescriptorsAndMessages(DESCRIPTOR, {modname!r}, _globals)
'''


def _module_for(proto_path):
    return proto_path[:-len(".proto")].replace("/", ".") + "_pb2"


def emit(root=ROOT):
    written = []
    for fd in build_files():
        imports = []
        for dep in fd.dependency:
            mod = _module_for(dep)
            pkg, leaf = mod.rsplit(".", 1)
            imports.append("from %s import %s as %s  # noqa: F401" % (pkg, leaf, mod.replace(".", "_dot_")))
        text = _HEADER.format(src=fd.name, imports="\n".join(imports), blob=fd.SerializeToString(),
                              modname=_module_for(fd.name))
        rel = fd.name[:-len(".proto")] + "_pb2.py"
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        # package markers down the tree
        d = os.path.dirname(path)
        while os.path.abspath(d) != os.path.abspath(root):
            init = os.path.join(d, "__init__.py")
            if not os.path.exists(init):
                open(init, "w").close()
            d = os.path.dirname(d)
        with open(path, "w") as fh:
            fh.write(text)
        written.append(path)
    return written


if __name__ == "__main__":
    for p in emit():
        sys.stdout.write(p + "\n")
