# -*- coding: utf-8 -*-
# Schema module written by tools/gen_pb2.py (no protoc in this image).  DO NOT EDIT BY HAND.
# source: tensorflow_serving/apis/inference.proto
"""Message classes for ``tensorflow_serving/apis/inference.proto`` built from a serialised FileDescriptorProto."""
from google.protobuf import descriptor_pool as _descriptor_pool
from google.protobuf import symbol_database as _symbol_database
from google.protobuf.internal import builder as _builder
from tensorflow_serving.apis import classification_pb2 as tensorflow_serving_dot_apis_dot_classification_pb2  # noqa: F401
from tensorflow_serving.apis import input_pb2 as tensorflow_serving_dot_apis_dot_input_pb2  # noqa: F401
from tensorflow_serving.apis import model_pb2 as tensorflow_serving_dot_apis_dot_model_pb2  # noqa: F401
from tensorflow_serving.apis import regression_pb2 as tensorflow_serving_dot_apis_dot_regression_pb2  # noqa: F401
_sym_db = _symbol_database.Default()

DESCRIPTOR = _descriptor_pool.Default().AddSerializedFile(b'\n\'tensorflow_serving/apis/inference.proto\x12\x12tensorflow.serving\x1a,tensorflow_serving/apis/classification.proto\x1a#tensorflow_serving/apis/input.proto\x1a#tensorflow_serving/apis/model.proto\x1a(tensorflow_serving/apis/regression.proto"n\n\rInferenceTask\x12<\n\nmodel_spec\x18\x01 \x01(\x0b2\x1d.tensorflow.serving.ModelSpecR\tmodelSpec\x12\x1f\n\x0bmethod_name\x18\x02 \x01(\tR\nmethodName"\x8f\x02\n\x0fInferenceResult\x12<\n\nmodel_spec\x18\x01 \x01(\x0b2\x1d.tensorflow.serving.ModelSpecR\tmodelSpec\x12_\n\x15classification_result\x18\x02 \x01(\x0b2(.tensorflow.serving.ClassificationResultH\x00R\x14classificationResult\x12S\n\x11regression_result\x18\x03 \x01(\x0b2$.tensorflow.serving.RegressionResultH\x00R\x10regressionResultB\x08\n\x06result"\x81\x01\n\x15MultiInferenceRequest\x127\n\x05tasks\x18\x01 \x03(\x0b2!.tensorflow.serving.InferenceTaskR\x05tasks\x12/\n\x05input\x18\x02 \x01(\x0b2\x19.tensorflow.serving.InputR\x05input"W\n\x16MultiInferenceResponse\x12=\n\x07results\x18\x01 \x03(\x0b2#.tensorflow.serving.InferenceResultR\x07resultsb\x06proto3')

_globals = globals()
_builder.BuildMessageAndEnumDescriptors(DESCRIPTOR, _globals)
_builder.BuildTopDescriptorsAndMessages(DESCRIPTOR, 'tensorflow_serving.apis.inference_pb2', _globals)
