"""Writes named arrays as an MXNet 1.x `.params` file in the layout crazyara_b200/mx_import.py reads (NDArray::Save of a
named list, V2 arrays, dense, on the CPU context) -- TEST INFRASTRUCTURE ONLY, for tests/test_mx_import.py.

style "prefixed" names the BatchNorm moving statistics `aux:<name>` and everything else `arg:<name>` (save_checkpoint,
HybridBlock.export); "bare" writes the names as they are (save_parameters).  dtype float32 or float16."""
import struct

import numpy as np

TYPE_FLAGS = {"float32": 0, "float64": 1, "float16": 2}


def array_record(a, dtype="float32", magic=0xF993FAC9, stype=0):
    a = np.ascontiguousarray(a, dtype=np.dtype(dtype).newbyteorder("<"))
    return (struct.pack("<Ii", magic, stype) + struct.pack(f"<I{a.ndim}q", a.ndim, *a.shape) +
            struct.pack("<iii", 1, 0, TYPE_FLAGS[dtype]) + a.tobytes())


def params_bytes(arrays, style="prefixed", dtype="float32", records=None):
    """-> the file's bytes; records replaces the array records (for files the reader must refuse)"""
    names = list(arrays)
    if style == "prefixed":
        names = [("aux:" if n.endswith(("_moving_mean", "_moving_var")) else "arg:") + n for n in names]
    records = records if records is not None else [array_record(a, dtype) for a in arrays.values()]
    head = struct.pack("<QQQ", 0x112, 0, len(records))
    return b"".join([head, *records, struct.pack("<Q", len(names))] +
                    [struct.pack("<Q", len(n.encode())) + n.encode() for n in names])


def write_params(arrays, path, style="prefixed", dtype="float32"):
    with open(path, "wb") as f:
        f.write(params_bytes(arrays, style, dtype))
    return path
