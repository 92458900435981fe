"""String MIN / MAX / COUNT and ANY of AggregateHash on the CPU (test infrastructure).

Groups, their order and the representative RowIDs come from the oracle (oracle_lib): string MIN / MAX / COUNT run there
as COUNT(*), and ANY is left out (an all-ANY query is the group-by-only call, the reference's DISTINCT path,
aggregate_hash.cpp:550-553, :1024-1061, :1209-1217), since the set of groups does not depend on the aggregates. This
module then computes, per group and in the reference's input order, MIN / MAX / COUNT of the string column with Python
bytes (they compare as unsigned bytes with a proper prefix first, as char_traits<char>::compare does), and ANY as the
column at the group's representative RowID (write_groupby_output, :421-537).
"""
import numpy as np

import aggregate_distinct_oracle as dorc
import oracle_lib as orc
from helpers import column_values_at
from hyrise_b200 import capi
from hyrise_b200.device import Aggregate

STRING_FUNCTIONS = (capi.AGG_MIN, capi.AGG_MAX, capi.AGG_COUNT)


def is_string_aggregate(table, aggregate) -> bool:
    return (aggregate.function in STRING_FUNCTIONS and aggregate.expression is not None
            and table.column_definitions[aggregate.expression.nodes[0][1]].data_type == capi.TYPE_STRING)


def _raw_strings(table, column_id):
    """Per row: the string as bytes (None for NULL), in chunk order."""
    out = []
    for chunk in table.chunks:
        segment = chunk.segments[column_id]
        out += [None if null else bytes(value) for value, null in zip(segment.decode(), segment.null_mask())]
    return out


def aggregate_hash(table, groupby_column_ids, aggregates, predicates=(), input_filter=None):
    """The reference's result: an AggregateOutput whose string MIN / MAX columns hold bytes (None for NULL), COUNT
    int64, and ANY the column at the representative RowIDs (Python values, None for NULL)."""
    placeholder = [Aggregate(capi.AGG_COUNT_STAR) if is_string_aggregate(table, a) else a
                   for a in aggregates if a.function != capi.AGG_ANY]
    output = orc.aggregate_hash(table, groupby_column_ids, placeholder, predicates=predicates, input_filter=input_filter)
    positions = dorc._positions(table, dorc.input_row_ids(table, predicates, input_filter))
    group_columns = [table.column_values(column_id) for column_id in groupby_column_ids]

    def keys_at(at):
        return list(zip(*[[None if n else v for v, n in zip(values[at].tolist(), nulls[at].tolist())]
                          for values, nulls in group_columns])) if group_columns else [()] * len(at)

    group_of_key = {}
    if len(positions) and output.group_count:
        group_of_key = {key: g for g, key in enumerate(keys_at(dorc._positions(table, output.row_ids)))}
    row_groups = [group_of_key.get(key, 0) for key in keys_at(positions)]

    values, nulls, types = [], [], []
    others = iter(zip(output.values, output.nulls, output.value_types))
    for aggregate in aggregates:
        if aggregate.function == capi.AGG_ANY:
            column_id = aggregate.expression.nodes[0][1]
            cells = column_values_at(table, column_id, output.row_ids) if output.group_count else []
            values.append(cells)
            nulls.append(np.array([cell is None for cell in cells], dtype=bool))
            types.append(table.column_definitions[column_id].data_type)
            continue
        value, null, value_type = next(others)
        if not is_string_aggregate(table, aggregate):
            values.append(value)
            nulls.append(null)
            types.append(value_type)
            continue
        strings = _raw_strings(table, aggregate.expression.nodes[0][1])
        per_group = [[] for _ in range(output.group_count)]
        for position, group in zip(positions.tolist(), row_groups):
            if strings[position] is not None:
                per_group[group].append(strings[position])
        if aggregate.function == capi.AGG_COUNT:
            values.append(np.array([len(entries) for entries in per_group], dtype=np.int64))
            nulls.append(np.zeros(output.group_count, dtype=bool))
            types.append(capi.TYPE_INT64)
        else:
            pick = min if aggregate.function == capi.AGG_MIN else max
            values.append([pick(entries) if entries else None for entries in per_group])
            nulls.append(np.array([not entries for entries in per_group], dtype=bool))
            types.append(capi.TYPE_STRING)
    output.values, output.nulls, output.value_types = values, nulls, types
    return output


def rows(table, groupby_column_ids, output) -> list[tuple]:
    """Result rows: the group-by values through the representative RowIDs, then each aggregate's Python value."""
    group_values = [column_values_at(table, column_id, output.row_ids) if output.group_count else []
                    for column_id in groupby_column_ids]
    out = []
    for g in range(output.group_count):
        row = [values[g] for values in group_values]
        for values, nulls in zip(output.values, output.nulls):
            cell = None if nulls[g] else values[g]
            row.append(cell.item() if hasattr(cell, "item") else cell)
        out.append(tuple(row))
    return out
