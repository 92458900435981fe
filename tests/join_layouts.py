"""Join inputs that pin JoinHash to one table kind and one family of probe kernels each, and a model of that choice.

Every builder returns a `JoinLayout`: build and probe tables, optional PosList inputs, and the facts the layout
guarantees — segment claims (chunk sizes, encodings, FoR offset widths), key facts (span, constant low bits, strictly
increasing, duplicates) and the hyb_join_path code an Inner join reports under each `TABLE_KINDS` setting. test_join_layouts.py checks all of them on
the host segments, so an encoder change fails there instead of moving a GPU case to other kernels unnoticed.

`predict_path` restates the table / kernel choice of hyb_join_hash (join.cu, `plan_join_table` and `plan_probe`)
from those facts; test_gpu_join_paths.py asserts the hyb_join_path code the library reports against it.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

import oracle_lib as orc
from aggregate_layouts import Claim, Layout, check_claims, table_from_chunks
from helpers import NULL_ROW
from hyrise_b200 import capi
from hyrise_b200.storage import ColumnDefinition, Table

I32, I64 = capi.TYPE_INT32, capi.TYPE_INT64
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SENTINEL = -0x7F7F7F7F7F7F7F80   # 0x8080808080808080: the int64 whose bytes are all 0x80
MODES = [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_SEMI, capi.JOIN_ANTI_NULL_AS_TRUE,
         capi.JOIN_ANTI_NULL_AS_FALSE]

# The five settings every GPU join case runs under (test_gpu_join.py, test_gpu_join_paths.py): (join_table, join_span,
# join_rank)
TABLE_KINDS = {"auto": ("auto", "1", "ballot"), "hash": ("hash", "1", "ballot"), "direct": ("direct", "1", "ballot"),
               "direct-tiles": ("direct", "0", "ballot"), "rank-match": ("rank", "1", "match")}
RANK, DIRECT, SHIFTED, HASH, HASH_WIDE = (capi.JOIN_PATH_TABLE_RANK, capi.JOIN_PATH_TABLE_DIRECT,
                                          capi.JOIN_PATH_TABLE_DIRECT_SHIFTED, capi.JOIN_PATH_TABLE_HASH,
                                          capi.JOIN_PATH_TABLE_HASH_WIDE)
SPAN_ROWS = 8192
SPAN, TILE_LEAN, TILE, RERUN = (capi.JOIN_PATH_PROBE_SPAN, capi.JOIN_PATH_PROBE_TILE_LEAN, capi.JOIN_PATH_PROBE_TILE,
                                capi.JOIN_PATH_RERUN)
# Every code a join can report (include/hyrise_b200.h names the combinations that cannot occur). With no probe rows the
# code is the table kind alone.
REACHABLE_PATHS = ({RANK, DIRECT, SHIFTED, HASH, HASH_WIDE} | {RANK | SPAN, RANK | TILE} |
                   {table | probe | rerun for table in (DIRECT, SHIFTED) for probe in (SPAN, TILE_LEAN, TILE)
                    for rerun in (0, RERUN)} |
                   {table | TILE | rerun for table in (HASH, HASH_WIDE) for rerun in (0, RERUN)})


# ---------------------------------------------------------------------------------------------------------------------
# PosList inputs
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class JoinFilter:
    """A PosList input: one side of a LEFT join (build side 0 holds NULL_ROW_IDs for unmatched probe rows, probe side 1
    the probe rows with NULL keys), or an ascending TableScan (`predicate`)."""
    source: str                      # "left-join" | "scan"
    table: Table | None = None       # left-join: the other table (probe of that join when this side is its build)
    side: int = 0                    # left-join: which side of the join result becomes the PosList
    predicate: object = None         # scan

    def host(self, this: Table, column: int) -> orc.HostPosList:
        if self.source == "scan":
            return orc.table_scan(this, self.predicate)
        build, probe = (this, self.table) if self.side == 0 else (self.table, this)
        result = orc.join_hash(build, column, probe, column, capi.JOIN_LEFT, 0)
        rows = result.build if self.side == 0 else result.probe
        # one slice holding the whole list: the join reads it in list order, as one PosList over many chunks
        return orc.HostPosList(rows, np.array([0] + [len(rows)] * this.chunk_count, dtype=np.uint64),
                               multiple_chunks=True)


# ---------------------------------------------------------------------------------------------------------------------
# Layouts
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class JoinLayout:
    name: str
    build: Table
    probe: Table
    build_claims: list
    probe_claims: list
    keys: dict                       # claimed facts of the build keys: span, low_bits, increasing, duplicates
    inner_paths: dict                # TABLE_KINDS setting -> the hyb_join_path code of an Inner join
    build_filter: JoinFilter | None = None
    probe_filter: JoinFilter | None = None
    column: int = 0
    extra: dict = field(default_factory=dict)


def paths(auto, hash_, direct, tiles, rank) -> dict:
    """Claimed Inner-join path per setting: auto, hash, direct, direct-tiles, rank-match."""
    return {"auto": auto, "hash": hash_, "direct": direct, "direct-tiles": tiles, "rank-match": rank}


# a strictly increasing dense int32 build, unfiltered int32 probe of lean codecs: rank + span kernels, or a direct
# table; a forced hash table takes the tile kernels
RANK_SPAN = paths(RANK | SPAN, HASH | TILE, DIRECT | SPAN, DIRECT | TILE_LEAN, RANK | SPAN)
# the same build against int64 probe keys: the rank table takes the generic loop, the direct table the int64 span path
RANK_WIDE = paths(RANK | TILE, HASH_WIDE | TILE, DIRECT | SPAN, DIRECT | TILE_LEAN, RANK | TILE)
# a dense int32 build with duplicate keys: a direct table, then the rerun
DIRECT_DUPLICATES = paths(DIRECT | SPAN | RERUN, HASH | TILE | RERUN, DIRECT | SPAN | RERUN,
                          DIRECT | TILE_LEAN | RERUN, DIRECT | SPAN | RERUN)
# a dense unique int32 build that is not increasing, probed through a PosList: the span kernels take no PosList
FILTERED_PROBE = paths(DIRECT | TILE_LEAN, HASH | TILE, DIRECT | TILE_LEAN, DIRECT | TILE_LEAN, DIRECT | TILE_LEAN)


def chunk_claims(text, sizes, encodings=None, vectors=None, nulls=None) -> list:
    """Claims per chunk: sizes, and where given the encoding / FixedWidth vector type / NULL mask of column 0."""
    claims = [Claim(f"{text}: chunk sizes {list(sizes)}", None, None, {"chunk_sizes": tuple(sizes)})]
    for chunk, _ in enumerate(sizes):
        checks = {}
        if encodings is not None:
            checks["encoding"] = encodings[chunk]
        if vectors is not None and vectors[chunk] is not None:
            checks["vector_type"] = vectors[chunk]
        if nulls is not None:
            checks["has_null_mask"] = nulls[chunk]
        if checks:
            claims.append(Claim(f"{text}: chunk {chunk} {checks}", 0, (chunk,), checks))
    return claims


def one_column(data_type, keys, chunk_sizes, encodings, nulls=None) -> Table:
    definition = ColumnDefinition("k", data_type, nulls is not None)
    keys = np.asarray(keys, dtype=np.int32 if data_type == I32 else np.int64)
    return table_from_chunks([definition], [keys], list(chunk_sizes), encodings, None if nulls is None else [nulls])


def per_chunk_encoded(data_type, keys, chunk_sizes, encodings) -> Table:
    """Chunk c encoded with encodings[c]."""
    table = one_column(data_type, keys, chunk_sizes, "Unencoded")
    for chunk, encoding in enumerate(encodings):
        table.encode(encoding, [chunk])
    return table


def dense_unique(rng, count, low, spread=2) -> np.ndarray:
    """`count` strictly increasing keys from [low, low + spread * count) that include odd and even keys."""
    keys = np.sort(rng.choice(spread * count, count, replace=False)) + low
    assert (keys & 1).any() and not (keys & 1).all()
    return keys


ENC = {"Unencoded": capi.ENC_UNENCODED, "FrameOfReference": capi.ENC_FRAME_OF_REFERENCE, "Dictionary": capi.ENC_DICTIONARY}
FOR_WIDTH = {1: capi.VEC_FIXED_1B, 2: capi.VEC_FIXED_2B, 4: capi.VEC_FIXED_4B}


# ---- 1. span codec matrix --------------------------------------------------------------------------------------------
SPAN_CHUNKS = (2 * SPAN_ROWS, 2 * SPAN_ROWS + 1, 511, 513, 65_535)   # full spans, one-row tail, partial only, 7 full + tail


def probe_chunk_keys(rng, codec, size, low, high) -> np.ndarray:
    """Probe keys of one chunk whose encoding gives `codec`: FoR offsets of 1 / 2 / 4 bytes, or plain values. Hits and
    misses on both sides of the build range [low, high)."""
    blocks = (size + capi.FOR_BLOCK_SIZE - 1) // capi.FOR_BLOCK_SIZE
    if codec == "for1":   # each 2048-row block within 256 keys of its own base
        base = rng.integers(low - 100, high - 100, blocks)
        return np.repeat(base, capi.FOR_BLOCK_SIZE)[:size] + rng.integers(0, 256, size)
    if codec == "for2":   # the build range +- 300 spans fewer than 2^16 keys
        return rng.integers(low - 300, high + 300, size)
    keys = rng.integers(low - 300, high + 300, size)   # for4, plain32, plain64: plus far misses
    keys[rng.random(size) < 0.01] = low - 5_000_000
    keys[0] = low - 5_000_000
    return keys


def span_codecs(codec: str) -> JoinLayout:
    """A strictly increasing dense int32 build (rank table under auto) against a probe whose every chunk decodes with one
    lean codec; chunks give full and partial 8192-row spans. `mixed` varies the codec by chunk."""
    rng = np.random.default_rng({"for1": 1, "for2": 2, "for4": 3, "plain32": 4, "plain64": 5, "mixed": 6}[codec])
    build_keys = dense_unique(rng, 30_000, 1_000)
    low, high = int(build_keys[0]), int(build_keys[-1]) + 1
    codecs = ["for1", "plain32", "for2", "for4", "for1"] if codec == "mixed" else [codec] * len(SPAN_CHUNKS)
    probe_type = I64 if codec == "plain64" else I32
    keys = np.concatenate([probe_chunk_keys(rng, c, size, low, high) for c, size in zip(codecs, SPAN_CHUNKS)])
    encodings = ["Unencoded" if c.startswith("plain") else "FrameOfReference" for c in codecs]
    if probe_type == I64:
        keys[::97] += 1 << 32   # same low 32 bits as a build key: must not match
    probe = per_chunk_encoded(probe_type, keys, SPAN_CHUNKS, encodings)
    vectors = [FOR_WIDTH[int(c[3])] if c.startswith("for") else None for c in codecs]
    build = one_column(I32, build_keys, [7_000, 7_000, 7_000, 7_000, 2_000], "Unencoded")
    wide = probe_type == I64
    return JoinLayout(
        f"span_{codec}", build, probe,
        chunk_claims("build", [7_000] * 4 + [2_000], [capi.ENC_UNENCODED] * 5),
        chunk_claims("probe", SPAN_CHUNKS, [ENC[e] for e in encodings], vectors, [False] * len(SPAN_CHUNKS)),
        {"span": high - 1 - low, "low_bits": 0, "increasing": True, "duplicates": False},
        RANK_WIDE if wide else RANK_SPAN)


def span_shifted_int64() -> JoinLayout:
    """int64 keys that agree in their 3 low bits (one rank's share of a radix exchange): a direct table indexed by
    (key - min) >> 3, probed by the span kernels with int64 keys; probe keys with other low bits must miss."""
    rng = np.random.default_rng(7)
    base = 7_000_000_000 + 5
    build_keys = base + 8 * dense_unique(rng, 20_000, 0)
    probe_keys = base + rng.integers(-400, 8 * 40_400, sum(SPAN_CHUNKS))
    probe_keys[::3] = base + 8 * rng.integers(-50, 40_050, len(probe_keys[::3]))   # low bits right: hits and misses
    build = one_column(I64, build_keys, [20_000], "Unencoded")
    probe = one_column(I64, probe_keys, SPAN_CHUNKS, "Unencoded")
    return JoinLayout(
        "span_plain64_shifted", build, probe,
        chunk_claims("build", [20_000], [capi.ENC_UNENCODED]),
        chunk_claims("probe", SPAN_CHUNKS, [capi.ENC_UNENCODED] * 5, None, [False] * 5),
        {"span": int(build_keys[-1] - build_keys[0]), "low_bits": 3, "increasing": True, "duplicates": False},
        paths(RANK | TILE, HASH_WIDE | TILE, SHIFTED | SPAN, SHIFTED | TILE_LEAN, RANK | TILE))


# ---- 2. int32 extremes -----------------------------------------------------------------------------------------------
def extreme_probe(rng, low, high) -> np.ndarray:
    """Both int32 ends, the build's min - 1 and max + 1 (where representable), and keys around the build range."""
    edges = [INT32_MIN, INT32_MIN + 1, INT32_MAX, INT32_MAX - 1, low, high]
    edges += [v for v in (low - 1, high + 1) if INT32_MIN <= v <= INT32_MAX]
    around = rng.integers(max(INT32_MIN, low - 500), min(INT32_MAX, high + 500) + 1, 6_000 - len(edges))
    keys = np.concatenate([np.array(edges, dtype=np.int64), around])
    return np.concatenate([keys, rng.permutation(keys)])


def int32_extreme(which: str) -> JoinLayout:
    """A dense build just below INT32_MAX (`top`) or just above INT32_MIN (`bottom`) — the lean paths compute
    key - min in wrapping 32-bit arithmetic — or a sparse build holding both ends (`both`), which only a hash table
    can hold. Probes: one plain and one FoR chunk with the same keys."""
    rng = np.random.default_rng({"top": 11, "bottom": 12, "both": 13}[which])
    if which == "top":
        build_keys = INT32_MAX - 19_999 + dense_unique(rng, 10_000, 0)
        build_keys[-1] = INT32_MAX
    elif which == "bottom":
        build_keys = INT32_MIN + dense_unique(rng, 10_000, 0)
        build_keys[0] = INT32_MIN
    else:
        build_keys = np.concatenate([[INT32_MIN, INT32_MIN + 1], rng.integers(-1_000, 1_000, 2_000), [INT32_MAX - 1,
                                                                                                     INT32_MAX]])
    build_keys = np.asarray(build_keys, dtype=np.int64)
    low, high = int(build_keys.min()), int(build_keys.max())
    probe_keys = extreme_probe(rng, low, high)
    half = len(probe_keys) // 2
    probe = per_chunk_encoded(I32, probe_keys, [half, half], ["Unencoded", "FrameOfReference"])
    build = one_column(I32, build_keys, [len(build_keys)], "Unencoded")
    dense = which != "both"
    tables = RANK_SPAN if dense else {kind: HASH | TILE | RERUN for kind in TABLE_KINDS}
    return JoinLayout(
        f"int32_{which}", build, probe,
        chunk_claims("build", [len(build_keys)], [capi.ENC_UNENCODED]),
        chunk_claims("probe", [half, half], [capi.ENC_UNENCODED, capi.ENC_FRAME_OF_REFERENCE], [None, capi.VEC_FIXED_4B]),
        {"span": high - low, "low_bits": 0, "increasing": dense, "duplicates": not dense},
        tables)


# ---- 3. int64 low-bit collisions -------------------------------------------------------------------------------------
def int64_collisions(duplicated: bool) -> JoinLayout:
    """Build keys k + j * 2^32 for several j (equal low 32 bits: the hash table must verify the full key), and probe
    keys with the same low bits and another j, which are absent; plus INT64_MIN / INT64_MAX."""
    rng = np.random.default_rng(21 + duplicated)
    low = rng.choice(5_000, 1_500, replace=False).astype(np.int64)
    j = np.array([-3, -1, 0, 1, 2], dtype=np.int64)
    build_keys = (low[:, None] + (j[None, :] << 32)).ravel()
    build_keys = np.concatenate([build_keys, [INT64_MIN, INT64_MAX, INT64_MIN + 1]])
    if duplicated:
        build_keys = np.concatenate([build_keys, build_keys[rng.integers(0, len(build_keys), 2_000)]])
    build_keys = rng.permutation(build_keys)
    probe_keys = np.concatenate([low[rng.integers(0, len(low), 6_000)] + (rng.integers(-4, 4, 6_000) << 32),
                                 [INT64_MIN, INT64_MAX, INT64_MAX - 1, INT64_MIN + 2, 0]])
    build = one_column(I64, build_keys, [len(build_keys) // 2, len(build_keys) - len(build_keys) // 2], "Unencoded")
    probe = one_column(I64, probe_keys, [len(probe_keys)], "Unencoded")
    return JoinLayout(
        f"int64_collisions{'_duplicated' if duplicated else ''}", build, probe,
        chunk_claims("build", [len(build_keys) // 2, len(build_keys) - len(build_keys) // 2]),
        chunk_claims("probe", [len(probe_keys)]),
        {"span": (1 << 64) - 1, "low_bits": 0, "increasing": False, "duplicates": duplicated},
        {kind: HASH_WIDE | TILE | (RERUN if duplicated else 0) for kind in TABLE_KINDS})


def int32_build_int64_probe() -> JoinLayout:
    """A dense int32 build against int64 probe keys 2^32 + k and -2^32 + k, which must not match k."""
    rng = np.random.default_rng(23)
    build_keys = dense_unique(rng, 8_000, -4_000)
    picks = build_keys[rng.integers(0, len(build_keys), 12_000)].astype(np.int64)
    probe_keys = picks + (rng.integers(-1, 2, len(picks)) << 32)
    build = one_column(I32, build_keys, [8_000], "Unencoded")
    probe = one_column(I64, probe_keys, [4_000, 8_000], "Unencoded")
    return JoinLayout(
        "int32_build_int64_probe", build, probe,
        chunk_claims("build", [8_000]), chunk_claims("probe", [4_000, 8_000], [capi.ENC_UNENCODED] * 2, None, [False] * 2),
        {"span": int(build_keys[-1] - build_keys[0]), "low_bits": 0, "increasing": True, "duplicates": False},
        RANK_WIDE)


def sentinel_pair(order: str) -> JoinLayout:
    """Two build rows, one bucket: 0x8080808080808080 (all bytes 0x80) and 0x80808080, which agree in their low 32 bits.
    Both insertion orders; the probe asks for both keys and for neighbours with the same low bits."""
    pair = [SENTINEL, 0x80808080] if order == "sentinel_first" else [0x80808080, SENTINEL]
    probe_keys = [SENTINEL, 0x80808080, 0x80808080 + (1 << 32), SENTINEL + (1 << 32), 0x80808080 - (1 << 32), 7,
                  SENTINEL, 0x80808080]
    build = one_column(I64, pair, [2], "Unencoded")
    probe = one_column(I64, probe_keys, [len(probe_keys)], "Unencoded")
    return JoinLayout(
        f"int64_{order}", build, probe, chunk_claims("build", [2]), chunk_claims("probe", [len(probe_keys)]),
        {"span": 0x80808080 - SENTINEL, "low_bits": 16, "increasing": order == "sentinel_first", "duplicates": False},
        {kind: HASH_WIDE | TILE for kind in TABLE_KINDS})


# ---- 4. non-uniform chunks -------------------------------------------------------------------------------------------
def chunked_build(name: str, sizes, duplicated=False) -> JoinLayout:
    """Build RowIDs from positions: chunk sizes that are not uniform (binary search over the chunk starts) or uniform
    powers of two and 1 (the multiply-shift division's edge shifts). Strictly increasing unless `duplicated`."""
    rng = np.random.default_rng(sum(sizes) + duplicated)
    rows = sum(sizes)
    build_keys = dense_unique(rng, rows, 100)
    if duplicated:
        build_keys = rng.permutation(build_keys)
        build_keys[rng.integers(0, rows, rows // 10)] = build_keys[rng.integers(0, rows, rows // 10)]
    probe_keys = rng.integers(0, 2 * rows + 300, min(3 * rows, 60_000))
    build = one_column(I32, build_keys, sizes, "Unencoded")
    probe_sizes = [len(probe_keys) // 2, len(probe_keys) - len(probe_keys) // 2]
    probe = per_chunk_encoded(I32, probe_keys, probe_sizes, ["FrameOfReference", "Unencoded"])
    span = int(build_keys.max() - build_keys.min())
    if duplicated:
        tables = DIRECT_DUPLICATES
    else:
        tables = RANK_SPAN
    return JoinLayout(name, build, probe, chunk_claims("build", sizes), chunk_claims("probe", probe_sizes),
                      {"span": span, "low_bits": 0, "increasing": not duplicated,
                       "duplicates": duplicated and len(np.unique(build_keys)) < rows}, tables)


def chunks_non_uniform():
    return chunked_build("chunks_7000_3000_7000_65535", [7_000, 3_000, 7_000, 65_535])


def chunks_empty_middle():
    return chunked_build("chunks_empty_middle_duplicated", [5_000, 0, 4_000, 5_000], duplicated=True)


def chunks_small_first():
    return chunked_build("chunks_small_first", [1_000, 8_000, 8_000, 3_000])


def chunks_of_one():
    return chunked_build("chunks_of_1", [1] * 300)


def chunks_of_4096():
    return chunked_build("chunks_of_4096_duplicated", [4_096] * 6 + [1_000], duplicated=True)


def chunks_of_16384():
    return chunked_build("chunks_of_16384", [16_384] * 3 + [77])


# ---- 5. heavy duplicates ---------------------------------------------------------------------------------------------
def heavy_duplicates(repeats: int = 50_000, hits: int = 200) -> JoinLayout:
    """One build key repeated `repeats` times among unique keys (the per-key sort of its positions), hit by `hits` probe
    rows: repeats x hits output pairs for that key alone."""
    rng = np.random.default_rng(41)
    unique = dense_unique(rng, 20_000, 0)
    hot = int(unique[777])
    build_keys = rng.permutation(np.concatenate([unique, np.full(repeats - 1, hot)]))
    probe_keys = np.concatenate([rng.integers(-100, int(unique[-1]) + 100, 5_000), np.full(hits, hot)])
    probe_keys = rng.permutation(probe_keys)
    sizes = [len(build_keys) // 2, len(build_keys) - len(build_keys) // 2]
    build = one_column(I32, build_keys, sizes, "Unencoded")
    probe = one_column(I32, probe_keys, [len(probe_keys)], "FrameOfReference")
    return JoinLayout(
        f"heavy_duplicates_{repeats}", build, probe, chunk_claims("build", sizes), chunk_claims("probe", [len(probe_keys)]),
        {"span": int(unique[-1] - unique[0]), "low_bits": 0, "increasing": False, "duplicates": True},
        DIRECT_DUPLICATES, extra={"hot_pairs": repeats * hits})


def heavy_duplicates_small() -> JoinLayout:
    return heavy_duplicates(400, 40)


def shifted_duplicates() -> JoinLayout:
    """int32 keys 4k + 1 with duplicates: a shifted direct table (shift 2) that needs the position lists, probed with
    int64 keys (the only probe type the lean loop and the span kernels take against a shifted table)."""
    rng = np.random.default_rng(43)
    build_keys = 1 + 4 * rng.integers(0, 6_000, 9_000)
    probe_keys = rng.integers(-20, 4 * 6_000 + 20, 20_000) + (rng.integers(-1, 2, 20_000) << 32)
    build = one_column(I32, build_keys, [4_000, 5_000], "Unencoded")
    probe = one_column(I64, probe_keys, [SPAN_ROWS + 1, 20_000 - SPAN_ROWS - 1], "Unencoded")
    return JoinLayout(
        "shifted_duplicates", build, probe, chunk_claims("build", [4_000, 5_000]),
        chunk_claims("probe", [SPAN_ROWS + 1, 20_000 - SPAN_ROWS - 1], [capi.ENC_UNENCODED] * 2, None, [False] * 2),
        {"span": int(build_keys.max() - build_keys.min()), "low_bits": 2, "increasing": False, "duplicates": True},
        paths(SHIFTED | SPAN | RERUN, HASH_WIDE | TILE | RERUN, SHIFTED | SPAN | RERUN, SHIFTED | TILE_LEAN | RERUN,
              SHIFTED | SPAN | RERUN))


# ---- 6. PosList inputs -----------------------------------------------------------------------------------------------
def poslist_tables(rng):
    base_keys = dense_unique(rng, 12_000, 0)
    nulls = rng.random(12_000) < 0.05
    base = one_column(I32, base_keys, [5_000, 5_000, 2_000], "Unencoded", nulls)
    other_keys = rng.integers(-100, int(base_keys[-1]) + 100, 9_000)
    other = one_column(I32, other_keys, [4_000, 5_000], "FrameOfReference")
    return base, other, base_keys[~nulls]


def poslist_left_build() -> JoinLayout:
    """The build-side PosList of a LEFT join (NULL_ROW_IDs for unmatched rows, in result order) as the build side."""
    rng = np.random.default_rng(51)
    base, other, base_keys = poslist_tables(rng)
    probe = one_column(I32, rng.integers(-50, int(base_keys[-1]) + 50, 10_000), [10_000], "FrameOfReference")
    return JoinLayout(
        "poslist_left_join_build", base, probe, chunk_claims("build", [5_000, 5_000, 2_000], nulls=[True] * 3),
        chunk_claims("probe", [10_000]),
        {"span": int(base_keys[-1] - base_keys[0]), "low_bits": 0, "increasing": False, "duplicates": True},
        DIRECT_DUPLICATES, build_filter=JoinFilter("left-join", other, side=0))


def poslist_left_probe() -> JoinLayout:
    """The same PosList (with NULL_ROW_IDs) as the probe side."""
    rng = np.random.default_rng(52)
    base, other, base_keys = poslist_tables(rng)
    build = one_column(I32, rng.permutation(base_keys)[:6_000], [6_000], "Unencoded")
    build_sorted = np.sort(np.asarray(build.column_values(0)[0], dtype=np.int64))
    return JoinLayout(
        "poslist_left_join_probe", build, base, chunk_claims("build", [6_000]),
        chunk_claims("probe", [5_000, 5_000, 2_000], nulls=[True] * 3),
        {"span": int(build_sorted[-1] - build_sorted[0]), "low_bits": 0, "increasing": False, "duplicates": False},
        FILTERED_PROBE, probe_filter=JoinFilter("left-join", other, side=0))


def poslist_left_probe_side() -> JoinLayout:
    """The probe-side PosList of a LEFT join as the probe side: its rows with NULL keys hold non-zero stored values and
    FoR placeholders, but a PosList over many chunks yields them as 0, which decides their partition."""
    rng = np.random.default_rng(54)
    keys = rng.integers(-3_000, 3_000, 12_000)
    nulls = rng.random(12_000) < 0.1
    probe = one_column(I32, keys, [5_000, 5_000, 2_000], "Unencoded", nulls)
    probe.encode("FrameOfReference", [1])
    build_keys = rng.permutation(np.arange(-2_000, 2_000))[:3_000]
    build = one_column(I32, build_keys, [3_000], "Unencoded")
    other = one_column(I32, rng.integers(-3_000, 3_000, 4_000), [4_000], "Unencoded")
    return JoinLayout(
        "poslist_left_join_probe_side", build, probe, chunk_claims("build", [3_000]),
        chunk_claims("probe", [5_000, 5_000, 2_000], [capi.ENC_UNENCODED, capi.ENC_FRAME_OF_REFERENCE, capi.ENC_UNENCODED],
                     nulls=[True] * 3),
        {"span": int(build_keys.max() - build_keys.min()), "low_bits": 0, "increasing": False, "duplicates": False},
        FILTERED_PROBE, probe_filter=JoinFilter("left-join", other, side=1))


def empty_probe(data_type) -> JoinLayout:
    """A probe PosList without rows (a scan that matches nothing): no probe kernel runs and the code is the table kind.
    int32 keys reach the rank, hash and direct tables; int64 keys 8k + 3 the wide hash and the shifted direct table."""
    from hyrise_b200.device import Predicate

    rng = np.random.default_rng(55)
    build_keys = dense_unique(rng, 5_000, 10)
    if data_type == I64:
        build_keys = (1 << 40) + 3 + 8 * build_keys
    build = one_column(data_type, build_keys, [5_000], "Unencoded")
    probe = one_column(data_type, build_keys[::-1], [3_000, 2_000], "Unencoded")
    wide = data_type == I64
    table = SHIFTED if wide else DIRECT
    return JoinLayout(
        f"empty_probe_{'int64' if wide else 'int32'}", build, probe, chunk_claims("build", [5_000]),
        chunk_claims("probe", [3_000, 2_000]),
        {"span": int(build_keys[-1] - build_keys[0]), "low_bits": 3 if wide else 0, "increasing": True,
         "duplicates": False},
        paths(RANK, HASH_WIDE if wide else HASH, table, table, RANK),
        probe_filter=JoinFilter("scan", predicate=Predicate(0, capi.PRED_LESS_THAN, int(build_keys[0]))))


def poslist_ascending_scan() -> JoinLayout:
    """An ascending TableScan over a strictly increasing column as the build side: the rank table still applies."""
    from hyrise_b200.device import Predicate

    rng = np.random.default_rng(53)
    build_keys = dense_unique(rng, 20_000, 0)
    build = one_column(I32, build_keys, [7_000, 7_000, 6_000], "Unencoded")
    probe = one_column(I32, rng.integers(-50, int(build_keys[-1]) + 50, 30_000), [30_000], "FrameOfReference")
    predicate = Predicate(0, capi.PRED_GREATER_THAN, int(build_keys[3_000]))
    return JoinLayout(
        "poslist_ascending_scan", build, probe, chunk_claims("build", [7_000, 7_000, 6_000]), chunk_claims("probe", [30_000]),
        {"span": int(build_keys[-1] - build_keys[0]), "low_bits": 0, "increasing": True, "duplicates": False},
        RANK_SPAN, build_filter=JoinFilter("scan", predicate=predicate))


# ---- 7. degenerate sides ---------------------------------------------------------------------------------------------
def all_null_build() -> JoinLayout:
    rng = np.random.default_rng(61)
    build = one_column(I32, np.zeros(3_000), [2_000, 1_000], "Unencoded", np.ones(3_000, dtype=bool))
    probe = one_column(I32, rng.integers(-10, 10, 5_000), [5_000], "Unencoded")
    return JoinLayout(
        "all_null_build", build, probe, chunk_claims("build", [2_000, 1_000], nulls=[True, True]), chunk_claims("probe", [5_000]),
        {"span": None, "low_bits": None, "increasing": False, "duplicates": False}, {kind: HASH | TILE for kind in TABLE_KINDS})


def one_row_build() -> JoinLayout:
    """One build row: every low bit is constant, so a forced direct table is a shifted one (shift 16)."""
    rng = np.random.default_rng(62)
    build = one_column(I32, [5], [1], "Unencoded")
    probe = one_column(I32, rng.integers(-3, 70_000, 6_000), [3_000, 3_000], "Unencoded", rng.random(6_000) < 0.1)
    probe.encode("FrameOfReference", [1])
    return JoinLayout(
        "one_row_build", build, probe, chunk_claims("build", [1]), chunk_claims("probe", [3_000, 3_000], nulls=[True, True]),
        {"span": 0, "low_bits": 16, "increasing": True, "duplicates": False},
        paths(RANK | TILE, HASH | TILE, SHIFTED | TILE, SHIFTED | TILE, RANK | TILE))


def all_null_probe() -> JoinLayout:
    rng = np.random.default_rng(63)
    build_keys = dense_unique(rng, 4_000, -2_000)
    build = one_column(I32, build_keys, [4_000], "Unencoded")
    probe = one_column(I32, np.zeros(5_000), [2_500, 2_500], "Unencoded", np.ones(5_000, dtype=bool))
    probe.encode("FrameOfReference", [1])
    return JoinLayout(
        "all_null_probe", build, probe, chunk_claims("build", [4_000]),
        chunk_claims("probe", [2_500, 2_500], [capi.ENC_UNENCODED, capi.ENC_FRAME_OF_REFERENCE], nulls=[True, True]),
        {"span": int(build_keys[-1] - build_keys[0]), "low_bits": 0, "increasing": True, "duplicates": False},
        paths(RANK | TILE, HASH | TILE, DIRECT | TILE_LEAN, DIRECT | TILE_LEAN, RANK | TILE))


def _span(codec):
    builder = lambda: span_codecs(codec)   # noqa: E731
    builder.__name__ = f"span_{codec}"
    return builder


def _named(name, function, *args):
    builder = lambda: function(*args)   # noqa: E731
    builder.__name__ = name
    return builder


# Every builder, in the sizes the GPU runs. heavy_duplicates (10^7 output pairs) is GPU-only; the CPU reference runs
# heavy_duplicates_small in its place.
BUILDERS = [_span(c) for c in ("for1", "for2", "for4", "plain32", "plain64", "mixed")] + [
    span_shifted_int64,
    _named("int32_top", int32_extreme, "top"), _named("int32_bottom", int32_extreme, "bottom"),
    _named("int32_both", int32_extreme, "both"),
    _named("int64_collisions", int64_collisions, False), _named("int64_collisions_duplicated", int64_collisions, True),
    int32_build_int64_probe,
    _named("int64_sentinel_first", sentinel_pair, "sentinel_first"), _named("int64_sentinel_last", sentinel_pair, "sentinel_last"),
    chunks_non_uniform, chunks_empty_middle, chunks_small_first, chunks_of_one, chunks_of_4096, chunks_of_16384,
    shifted_duplicates, poslist_left_build, poslist_left_probe, poslist_left_probe_side, poslist_ascending_scan,
    _named("empty_probe_int32", empty_probe, I32), _named("empty_probe_int64", empty_probe, I64),
    all_null_build, one_row_build, all_null_probe,
]
GPU_BUILDERS = BUILDERS + [heavy_duplicates]
CPU_BUILDERS = BUILDERS + [heavy_duplicates_small]


# ---------------------------------------------------------------------------------------------------------------------
# Host facts and the model of the path choice
# ---------------------------------------------------------------------------------------------------------------------
def side_rows(table: Table, column: int, pos_list: orc.HostPosList | None):
    """[(RowID tuple, key or None, NULL placeholder)] in position order. The placeholder is the value the reference's
    iterators yield for a NULL row, which decides its partition: the stored value of a ValueSegment, minimum + offset of
    a FrameOfReference segment, 0 for a dictionary, for a NULL_ROW_ID and for every NULL row of a PosList over many
    chunks (MultipleChunkIterator yields T{})."""
    decoded = []
    for chunk in table.chunks:
        segment = chunk.segments[column]
        values = segment.decode().astype(np.int64)
        nulls = segment.null_mask()
        if segment.encoding == capi.ENC_DICTIONARY:
            values = np.where(nulls, 0, values)
        decoded.append((values.tolist(), nulls.tolist()))
    if pos_list is None:
        positions = [(chunk_id, offset) for chunk_id, chunk in enumerate(table.chunks) for offset in range(chunk.size)]
    else:
        positions = [(int(r["chunk_id"]), int(r["chunk_offset"])) for r in pos_list.row_ids]
    out = []
    for row_id in positions:
        if row_id == NULL_ROW:
            out.append((row_id, None, 0))
            continue
        values, nulls = decoded[row_id[0]]
        value = values[row_id[1]]
        if not nulls[row_id[1]]:
            out.append((row_id, value, value))
        else:
            out.append((row_id, None, 0 if pos_list is not None and pos_list.multiple_chunks else value))
    return out


@dataclass
class SideFacts:
    data_type: int
    positions: int
    has_values: bool
    key_min: int
    key_max: int
    low_bits: int
    increasing: bool                 # the whole column, in table order, without a NULL
    duplicates: bool                 # among the side's non-NULL positions
    filtered: bool
    filter_ascending: bool
    span_codecs: bool                # every chunk: no NULL vector, not a dictionary, not bit-packed FoR


def side_facts(table: Table, column: int, pos_list: orc.HostPosList | None, ascending: bool) -> SideFacts:
    """What the library knows about one join side: the key bounds of the whole column (cached per column, so a PosList
    input shares them), and the positions, duplicates and codecs of the side itself."""
    values, nulls = table.column_values(column)
    values = values.astype(np.int64)
    keys = values[~nulls]
    low_bits = 0
    if len(keys):
        varying = int(np.bitwise_or.reduce(keys ^ keys[0])) & ((1 << 64) - 1)
        while low_bits < 16 and not (varying >> low_bits) & 1:
            low_bits += 1
    increasing = bool(len(keys)) and len(keys) == len(values) and bool(np.all(keys[1:] > keys[:-1]))
    if pos_list is None:
        positions, side_keys = len(values), keys
    else:
        rows = pos_list.row_ids
        real = rows["chunk_id"] != NULL_ROW[0]
        starts = np.cumsum([0] + [chunk.size for chunk in table.chunks])
        index = starts[rows["chunk_id"][real].astype(np.int64)] + rows["chunk_offset"][real].astype(np.int64)
        positions, side_keys = len(rows), values[index][~nulls[index]]
    span_codecs = all(s.nulls is None and s.encoding != capi.ENC_DICTIONARY and s.vector_type != capi.VEC_BITPACKED
                      for s in (chunk.segments[column] for chunk in table.chunks))
    return SideFacts(table.column_definitions[column].data_type, positions, bool(len(keys)),
                     int(keys.min()) if len(keys) else 0, int(keys.max()) if len(keys) else 0, low_bits, increasing,
                     len(np.unique(side_keys)) < len(side_keys), pos_list is not None, ascending, span_codecs)


def layout_facts(layout: JoinLayout, build_list=None, probe_list=None):
    ascending = layout.build_filter is not None and layout.build_filter.source == "scan"
    return (side_facts(layout.build, layout.column, build_list, ascending),
            side_facts(layout.probe, layout.column, probe_list, False))


def predict_table(build: SideFacts, probe: SideFacts, kind: str) -> tuple[int, int, bool, bool]:
    """(table code, direct shift, direct, rank) as plan_join_table chooses them."""
    table_option = TABLE_KINDS[kind][0]
    key_span = (build.key_max - build.key_min) & ((1 << 64) - 1)
    shift = build.low_bits
    direct_span = key_span >> shift
    direct = (build.has_values and build.positions > 0 and direct_span < 0xFFFFFFE0 and table_option != "hash" and
              (direct_span < 8 * build.positions + 65_536 or (table_option != "auto" and direct_span < (1 << 28))))
    rank = (direct and table_option != "direct" and build.increasing and key_span < 0xFFFFFFE0 and
            (not build.filtered or build.filter_ascending))
    wide = I64 in (build.data_type, probe.data_type)
    code = RANK if rank else (SHIFTED if shift else DIRECT) if direct else HASH_WIDE if wide else HASH
    return code, shift, direct, rank


def predict_path(build: SideFacts, probe: SideFacts, kind: str, mode: int) -> int:
    code, shift, direct, rank = predict_table(build, probe, kind)
    wide = I64 in (build.data_type, probe.data_type)
    fast = 0
    if mode == capi.JOIN_INNER and (direct or rank):
        fast = 1 if (shift == 0 and not wide) else (2 if (not rank and probe.data_type == I64) else 0)
    if probe.positions == 0:
        return code
    span = (TABLE_KINDS[kind][1] == "1" and fast != 0 and not probe.filtered and probe.span_codecs and
            ((fast == 2) == (probe.data_type == I64)))
    tile_fast = fast != 0 and not rank
    code |= (capi.JOIN_PATH_PROBE_SPAN if span else capi.JOIN_PATH_PROBE_TILE_LEAN if tile_fast else
             capi.JOIN_PATH_PROBE_TILE)
    semi_or_anti = mode in (capi.JOIN_SEMI, capi.JOIN_ANTI_NULL_AS_TRUE, capi.JOIN_ANTI_NULL_AS_FALSE)
    if build.duplicates and not rank and not semi_or_anti:
        code |= capi.JOIN_PATH_RERUN
    return code


def check_layout(layout: JoinLayout) -> None:
    """Every claim of a builder against its host segments, and the table kind of every setting against the model."""
    check_claims(Layout(layout.name + " build", layout.build, layout.build_claims))
    check_claims(Layout(layout.name + " probe", layout.probe, layout.probe_claims))
    build_list = layout.build_filter.host(layout.build, layout.column) if layout.build_filter else None
    probe_list = layout.probe_filter.host(layout.probe, layout.column) if layout.probe_filter else None
    build, probe = layout_facts(layout, build_list, probe_list)
    claimed = layout.keys
    if claimed["span"] is not None:
        assert (build.key_max - build.key_min) & ((1 << 64) - 1) == claimed["span"] % (1 << 64), layout.name
        assert build.low_bits == claimed["low_bits"], (layout.name, build.low_bits)
    assert build.has_values == (claimed["span"] is not None), layout.name
    assert build.increasing == claimed["increasing"], layout.name
    assert build.duplicates == claimed["duplicates"], layout.name
    for kind, want in layout.inner_paths.items():
        assert predict_path(build, probe, kind, capi.JOIN_INNER) == want, (layout.name, kind)
    assert set(layout.inner_paths) == set(TABLE_KINDS)


def reference_output(layout: JoinLayout, mode: int, radix_bits: int, build_list=None, probe_list=None):
    """helpers.reference_join_order on the decoded sides: the exact output sequence, as RowID tuples."""
    from helpers import reference_join_order

    build_rows = [(row_id, key) for row_id, key, _ in side_rows(layout.build, layout.column, build_list)]
    probe_rows = side_rows(layout.probe, layout.column, probe_list)
    return reference_join_order(build_rows, probe_rows, mode, radix_bits)
