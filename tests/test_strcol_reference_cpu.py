"""tests/strcol_ref.py against the protobuf runtime and the protobuf-backed definitions, and its geometry model against the sources
(no GPU)."""
import numpy as np
import pytest

import example_ref as E
import padded_string_decode_ref as PR
import padded_strings_ref as PS
import strcol_ref as S
import string_responses as SR
from min_tfs_client.codec import BytesColumn, RaggedColumn
from min_tfs_client.requests import TensorServingClient, examples_from_input_dict, examples_with_context_from_input_dict
from tensorflow.core.framework import types_pb2
from tensorflow_serving.apis.classification_pb2 import ClassificationRequest
from tensorflow_serving.apis.predict_pb2 import PredictRequest

LENS = [0, 1, 15, 16, 17, 63, 64, 65, 127, 128, 16383, 16384, 16385, (1 << 21) - 1, 1 << 21]


def corpus(seed=0):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in LENS] + [b"\x00" * 3, b"\xff\x80\x00"]


def bytes_column(strs, shape, start=0):
    off = np.r_[0, np.cumsum(S.lens_of(strs))].astype(np.int64) + start
    return BytesColumn(np.concatenate([np.full(start, 0xEE, np.uint8), S.flat_of(strs), np.zeros(2, np.uint8)]), off, shape)


def test_constants_are_the_sources_literals():
    assert (S.K_LANE, S.K_BLOCK, S.K_CHUNK, S.K_STR_THREADS) == (64, 16384, 256, 256)
    assert (S.K_VAR_THREADS, S.K_GROUP_TILES, S.K_STAGE, S.LINE) == (256, 256, 16384, 128)
    assert "line = a >> 7" in E._source("walker.h")          # rd8's line number agrees with the 128-byte rounding


@pytest.mark.parametrize("dims", [(17,), (1, 17), (17, 1, 1)])
def test_string_val_tensor_and_request_match_the_runtime(dims):
    strs = corpus()
    tp = S.tensor_proto(S.string_val_body(strs), dims)
    assert tp == PS.string_proto(strs, dims).SerializeToString(deterministic=True)
    for inputs in ({"s": (strs, dims)}, {"b": (strs[:3], (3,)), "a": ([], (0, 4))}):
        protos = {k: S.tensor_proto(S.string_val_body(v[0]), v[1]) for k, v in inputs.items()}
        want = PS.request_wire("m", 3, {k: PS.string_proto(*v) for k, v in inputs.items()})
        assert S.predict_request("m", 3, protos) == want


def test_tiled_values_gather_like_the_list():
    strs = corpus()[:12]
    pattern = np.random.default_rng(1).integers(0, 12, 5000)
    sz, flat = S.tiled_values(strs, pattern, 0x42)
    assert flat.tobytes() == S.string_val_body([strs[i] for i in pattern])
    assert sz.tolist() == [S.string_values([strs[i]], 0x42)[0][0] for i in pattern]


def runtime_request(d, key, context=None):
    """what the protobuf runtime makes of the request: Classify (key None) or Predict, with an ExampleListWithContext when
    context is not None"""
    if key is None:
        return TensorServingClient._make_example_request(None, ClassificationRequest, "m", d, 1, context).SerializeToString(deterministic=True)
    msg = PredictRequest()
    msg.model_spec.name = "m"
    msg.model_spec.version.value = 1
    if context is None:
        values = examples_from_input_dict(d).example_list.examples
    else:
        values = [examples_with_context_from_input_dict(d, context).example_list_with_context]
    t = msg.inputs[key]
    t.dtype = types_pb2.DT_STRING
    t.tensor_shape.dim.add().size = len(values)
    t.string_val.extend(v.SerializeToString(deterministic=True) for v in values)
    return msg.SerializeToString(deterministic=True)


@pytest.mark.parametrize("m", [0, 31, 32, 33, 65])
def test_bytes_list_context_matches_the_runtime(m):
    rng = np.random.default_rng(m)
    strs = corpus()[:10]
    d = {"s": bytes_column([strs[i] for i in rng.integers(0, 10, 6)], (2, 3)), "x": np.ones((2, 1), np.float32)}
    ctx = {"c": bytes_column([strs[i] for i in rng.integers(0, 10, m)], None, start=3), "one": bytes_column([b"\x00q"], ()),
           "i": np.arange(4)}
    for key in (None, "elwc"):
        for c in (ctx, {}):
            assert E.request_bytes("m", 1, d, key=key, context=c) == runtime_request(d, key, c)


@pytest.mark.parametrize("width", [0, 31, 32, 33, 65])
def test_bytes_list_rows_match_the_runtime(width):
    rng = np.random.default_rng(width)
    strs = corpus()[:10]
    n = 3
    cells = [strs[i] for i in rng.integers(0, 10, n * width)]
    d = {"s": bytes_column(cells, (n, width), start=5), "one": bytes_column([b"\x00\xff"], ()), "x": np.ones((n, 2), np.float32),
         "r": RaggedColumn(bytes_column(cells[: n * width], (n, width)), np.array([0, width, width // 2]))}
    for key in (None, "examples"):
        assert E.request_bytes("m", 1, d, key=key) == runtime_request(d, key)
    assert S.example_rounds(width) == (-(-width // 32), max(-(-width // 32) - 1, 0))


def test_decode_columns_match_the_definitions():
    rng = np.random.default_rng(2)
    strs = corpus()[:12]
    parts = [[strs[i] for i in rng.integers(0, 12, k)] for k in (3, 0, 5, 1)]
    wires = [SR.response(("s", SR.string_tensor(p, [len(p)]))) for p in parts]
    data, off, _ = SR.reference(wires, "s")
    got = S.concat_column(parts)
    assert got[0].tobytes() == data.tobytes() and got[1].tolist() == off.tolist()
    pp = [(p, (1, len(p))) for p in parts]
    wires = [SR.response(("s", SR.string_tensor(p, [1, len(p)]))) for p in parts]
    for pad in (b"", b"<pad>"):
        data, off, shape, _ = PR.reference(wires, "s", pad)
        got = S.padded_column(pp, shape[1:], pad)
        assert got[0].tobytes() == data.tobytes() and got[1].tolist() == off.tolist()


def test_tiers_follow_warp_copy_strings():
    assert [S.tier(x) for x in (0, 64, 65, 16384, 16385)] == ["lane", "lane", "warp", "warp", "warp"]
    assert [S.tier(x, cta=True) for x in (64, 65, 16384, 16385)] == ["lane", "warp", "warp", "cta"]
    lens = [65 if i % 2 else 3 for i in range(32)] + [0] * 31 + [70]
    assert [S.lane_mix(m) for m, _ in S.warp_rounds(lens)] == ["alternating", "only_lane31"]


def test_tiles_and_chunks_partition_their_strings():
    for m in (0, 1, 255, 256, 257, 65536, 65537, 131073):
        j = S.EncodeJob(np.zeros(m, np.int64), np.arange(m))
        assert j.tiles == max(1, -(-m // 256)) and np.bincount(j.tile_of, minlength=j.tiles).sum() == m
        assert j.groups == -(-j.tiles // 256) and not j.crossing_tiles
    counts = np.array([[255, 0, 256, 257, 0], [0, 1, 0, 512, 3]])
    ok = np.ones_like(counts, bool)
    ok[1, 3] = False
    ch, c0, total = S.concat_chunks(counts, ok)
    owners = [S.pair_of(c0, c) for c in range(total)]
    assert sorted(owners) == sorted(q for q in range(len(ch)) for _ in range(ch[q]))
    assert set(S.tied_pairs(ch, c0)) >= {1, 5, 8}
    st, first, last = S.concat_scan([5, 0, 9, 0, 2], [True] * 5, 6)
    assert st == ["ok", "ok", "size", "size", "size"] and first == [0, 5, 5, 14, 14] and last == 5


def test_emit_plan_of_bytes_columns_follows_ex_layout():
    """ReqPlan sizes a bytes column as ex_layout does: no strings plus 27 bytes in ex_max, plus 18 for the example header, the
    strings' bound in the slot, the expected size for the spans"""
    strs = [b"a" * 100, b"", b"b" * 20000]
    col = bytes_column(strs, (3,), start=5)
    q = E.ReqPlan("m", 1, {"s": col})
    assert q.ex_max == E._example_len(E._bytes_entry_len(0, 1) + 27) + 18
    assert q.ex_expect == q.ex_max + 2 + col.data_len // 3 and q.per == max(1, E.K_STAGE // q.ex_expect)
    assert q.str_bound == 3 * 11 + col.data_len and q.counted and not q.has_int
    sizes, _ = E.example_bytes({"s": col})
    E.plan([q])
    assert E.covers_once(q, sizes, E.emit(q, sizes)["stores"])


def test_walk_lines_follow_the_address():
    f = S.string_fields(120, [200, 3])
    assert S.walk_lines(0, f)[0] == (0, 0, 0, 0) and S.walk_lines(7, f)[0] == (0, 1, 1, 1)
    assert S.crossing_varints(S.walk_lines(7, f)) == [0]
