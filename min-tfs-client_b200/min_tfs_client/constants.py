"""numpy <-> tensorflow.DataType <-> TensorProto field table.

Same rows, names and derived maps as the reference's ``min_tfs_client/constants.py:13-50`` (15 numpy
types), so code that imports these names keeps working.  ``BFLOAT16`` is an addition: the reference
rejects it (``ValueError`` from ``DataType``), TF stores it in ``half_val`` as bit patterns.
"""
from typing import NamedTuple

import numpy as np

from tensorflow.core.framework import types_pb2


class TFType(NamedTuple):
    TFDType: str
    TensorProtoField: str


_ROWS = (
    (np.float16, "DT_HALF", "half_val"),
    (np.float32, "DT_FLOAT", "float_val"),
    (np.float64, "DT_DOUBLE", "double_val"),
    (np.int8, "DT_INT8", "int_val"),
    (np.int16, "DT_INT16", "int_val"),
    (np.int32, "DT_INT32", "int_val"),
    (np.int64, "DT_INT64", "int64_val"),
    (np.uint8, "DT_UINT8", "int_val"),
    (np.uint16, "DT_UINT16", "int_val"),
    (np.uint32, "DT_UINT32", "uint32_val"),
    (np.uint64, "DT_UINT64", "uint64_val"),
    (np.complex64, "DT_COMPLEX64", "scomplex_val"),
    (np.complex128, "DT_COMPLEX128", "dcomplex_val"),
    (np.str_, "DT_STRING", "string_val"),
    (np.bool_, "DT_BOOL", "bool_val"),
)

NP_TO_TF_MAPPING = {np_type: TFType(TFDType=dt, TensorProtoField=field) for np_type, dt, field in _ROWS}
TF_TO_NP_MAPPING = {v.TFDType: k for k, v in NP_TO_TF_MAPPING.items()}
NP_TO_ENUM_MAPPING = {k: getattr(types_pb2, v.TFDType) for k, v in NP_TO_TF_MAPPING.items()}
ENUM_TO_TF_MAPPING = {v: NP_TO_TF_MAPPING[k].TFDType for k, v in NP_TO_ENUM_MAPPING.items()}

NUMERICAL_TYPES = {np_type for np_type, _, _ in _ROWS if np_type is not np.str_}

# --- additions for the GPU codec --------------------------------------------------------------
try:  # optional: bfloat16 host arrays
    import ml_dtypes as _ml_dtypes

    BFLOAT16 = _ml_dtypes.bfloat16
except ImportError:  # pragma: no cover
    BFLOAT16 = None

DT_BFLOAT16 = types_pb2.DT_BFLOAT16


def enum_for_numpy(np_dtype) -> int:
    """DT_* enum value for a numpy dtype (reference table + bfloat16); KeyError if unmapped."""
    t = np.dtype(np_dtype).type
    if BFLOAT16 is not None and t is BFLOAT16:
        return DT_BFLOAT16
    return NP_TO_ENUM_MAPPING[t]


def numpy_for_enum(enum: int):
    """numpy scalar type for a DT_* value (reference table + bfloat16); KeyError if unmapped."""
    if enum == DT_BFLOAT16 and BFLOAT16 is not None:
        return BFLOAT16
    return np.dtype(TF_TO_NP_MAPPING[ENUM_TO_TF_MAPPING[enum]]).type
