"""The table hyb_aggregate_result_table derives from an aggregate result, built on the host: an AGGREGATE column holds the
result's values and NULLs as they are, a COLUMN column the aggregated table's column read at each group's representative
RowID (a ReferenceSegment's reading; NULL at NULL_ROW_ID), chunked like the device table."""
from __future__ import annotations

import numpy as np

from helpers import column_values_at
from hyrise_b200 import capi
from hyrise_b200.storage import NUMPY_TYPES, ColumnDefinition, Table


def expected_table(source: Table, output, columns, chunk_size: int) -> Table:
    """`output`: an AggregateOutput of `source` (oracle_lib.aggregate_hash or the device's); `columns`: (kind, index)."""
    definitions, arrays, nulls = [], [], []
    valid_rows = output.row_ids["chunk_id"] != 0xFFFFFFFF  # NULL_ROW_ID: the synthesised row
    for kind, index in columns:
        if kind == capi.SORT_KEY_AGGREGATE:
            data_type = output.value_types[index]
            values = np.asarray(output.values[index], dtype=NUMPY_TYPES[data_type])
            null = np.asarray(output.nulls[index], dtype=bool)
            name = f"aggregate_{index}"
        else:
            definition = source.column_definitions[index]
            data_type, name = definition.data_type, definition.name
            dtype = NUMPY_TYPES.get(data_type, "S64")
            values = np.zeros(output.group_count, dtype=dtype)
            null = np.ones(output.group_count, dtype=bool)
            read = column_values_at(source, index, output.row_ids[valid_rows]) if valid_rows.any() else []
            for position, value in zip(np.flatnonzero(valid_rows), read):
                if value is not None:
                    values[position] = value
                    null[position] = False
        definitions.append(ColumnDefinition(name, data_type, True))
        arrays.append(values)
        nulls.append(null)
    return Table.from_columns(definitions, arrays, nulls, chunk_size)
