"""CPU tests of the PartialReduce aggregate ops: the header's dfd_agg_op values are the Python binding's AGG_* constants,
agg_op() maps every Arrow state type that has a device op and refuses the rest, and the library's k_group_combine holds
the 128-bit CAS the Decimal128 MIN / MAX is built on."""
import os
import re
import subprocess

import pyarrow as pa
import pytest

from datafusion_distributed_b200 import _native as nv
from datafusion_distributed_b200 import agg_op

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_agg_ops():
    text = open(os.path.join(ROOT, "include", "dfd_b200.h")).read()
    body = re.search(r"typedef enum \{([^}]*)\} dfd_agg_op;", text).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return {name: int(v) for name, v in re.findall(r"DFD_(AGG_[A-Z0-9_]+)\s*=\s*(\d+)", body)}


def test_header_agg_ops_equal_the_python_constants():
    ops = header_agg_ops()
    assert len(ops) == 27 and sorted(ops.values()) == list(range(27))
    assert ops == {name: getattr(nv, name) for name in dir(nv) if name.startswith("AGG_")}


MIN_MAX = [  # (state type, MIN op); MAX is the next value
    (pa.int64(), nv.AGG_MIN_I64), (pa.timestamp("ns"), nv.AGG_MIN_I64), (pa.timestamp("us", "UTC"), nv.AGG_MIN_I64),
    (pa.date64(), nv.AGG_MIN_I64), (pa.time64("ns"), nv.AGG_MIN_I64), (pa.duration("ms"), nv.AGG_MIN_I64),
    (pa.decimal64(18, 2), nv.AGG_MIN_I64),
    (pa.int32(), nv.AGG_MIN_I32), (pa.date32(), nv.AGG_MIN_I32), (pa.time32("s"), nv.AGG_MIN_I32), (pa.decimal32(9, 2), nv.AGG_MIN_I32),
    (pa.int16(), nv.AGG_MIN_I16), (pa.int8(), nv.AGG_MIN_I8),
    (pa.uint64(), nv.AGG_MIN_U64), (pa.uint32(), nv.AGG_MIN_U32), (pa.uint16(), nv.AGG_MIN_U16), (pa.uint8(), nv.AGG_MIN_U8),
    (pa.decimal128(15, 2), nv.AGG_MIN_I128), (pa.decimal128(38, 0), nv.AGG_MIN_I128),
    (pa.float64(), nv.AGG_MIN_F64), (pa.float32(), nv.AGG_MIN_F32), (pa.float16(), nv.AGG_MIN_F16),
]


@pytest.mark.parametrize("arrow_type,min_op", MIN_MAX, ids=[str(t) for t, _ in MIN_MAX])
def test_agg_op_min_max(arrow_type, min_op):
    assert agg_op(arrow_type, "min") == min_op
    assert agg_op(arrow_type, "max") == min_op + 1
    names = {v: k for k, v in header_agg_ops().items()}
    assert names[min_op].startswith("AGG_MIN_") and names[min_op + 1] == names[min_op].replace("MIN", "MAX")


def test_agg_op_sum():
    assert agg_op(pa.int64(), "sum") == nv.AGG_SUM_I64  # also COUNT states
    assert agg_op(pa.uint64(), "sum") == nv.AGG_SUM_I64
    assert agg_op(pa.float64(), "sum") == nv.AGG_SUM_F64
    assert agg_op(pa.decimal128(38, 4), "sum") == nv.AGG_SUM_I128
    for t in (pa.int32(), pa.float32(), pa.decimal64(18, 2), pa.string(), pa.bool_()):
        with pytest.raises(ValueError):
            agg_op(t, "sum")


REFUSED = [pa.string(), pa.large_string(), pa.string_view(), pa.binary(), pa.binary(16), pa.bool_(), pa.month_day_nano_interval(),
           pa.decimal256(40, 2), pa.list_(pa.int32()), pa.struct([("a", pa.int32())]), pa.dictionary(pa.int32(), pa.string()), pa.null()]


@pytest.mark.parametrize("arrow_type", REFUSED, ids=[str(t) for t in REFUSED])
def test_agg_op_refuses_states_without_a_device_op(arrow_type):
    for kind in ("min", "max"):
        with pytest.raises(ValueError):
            agg_op(arrow_type, kind)


def test_agg_op_refuses_unknown_kinds():
    with pytest.raises(ValueError):
        agg_op(pa.int64(), "avg")


def test_combine_kernel_holds_a_128_bit_cas(built):
    """The Decimal128 MIN / MAX compiles to one 16-byte CAS per attempt (no lock, no split 64-bit update)."""
    from datafusion_distributed_b200 import LIB_PATH

    sass = subprocess.run(["cuobjdump", "-sass", LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    combine = [f for f in funcs if f.split("\n", 1)[0].find("k_group_combine") >= 0]
    assert len(combine) == 1, [f.split("\n", 1)[0] for f in funcs if "k_group" in f.split("\n", 1)[0]]
    assert "ATOMG.E.CAS.128" in combine[0]
