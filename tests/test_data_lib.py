"""CPU: maro_b200.data_lib.BinaryConverter (SURVEY.md §8f rank 3) against the reference's own csv / bin fixture pairs
(reference tests/data/citi_bike, tests/data/vm_scheduling, tests/data/data_lib — the .bin files were written by the reference's
converter: either shipped next to the csv in its test data, or converted here by tests/golden/gen_bike_golden.py) — byte for byte —
and the round trip through the reader the scenario loaders use."""
import os

import numpy as np
import pytest

from maro_b200.data_lib import BinaryConverter, read_bin

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
D = os.path.join(G, "data_lib")

PAIRS = [
    # csv, meta, reference-written bin (relative to tests/golden: test ids must not depend on where the checkout lives)
    ("trips_case_1.csv", "trips.meta.yml", "bike_case_1/trips.bin"),
    ("trips_case_2.csv", "trips.meta.yml", "bike_case_2/trips.bin"),
    ("weather.csv", "weather.meta.yml", "bike_case_1/weathers.bin"),
    ("vmtable_toy.csv", "vmtable_toy.meta.yml", "vm_toy/vmtable_toy.bin"),
    ("vm_cpu_readings-file-1-of-toy.csv", "cpu_readings.yml", "vm_toy/vm_cpu_readings-file-1-of-toy.bin"),
    ("vmtable_test.csv", "vmtable.meta.yml", "data_lib/vmtable_test.bin"),
    ("vm_cpu_readings-file-2-of-test.csv", "cpu_readings.yml", "data_lib/vm_cpu_readings-file-2-of-test.bin"),
    ("vm_cpu_readings-file-1-of-test.csv", "cpu_readings.yml", "data_lib/vm_cpu_readings-file-1-of-test.bin"),
    ("vm_cpu_readings-file-3-of-test.csv", "cpu_readings.yml", "data_lib/vm_cpu_readings-file-3-of-test.bin"),
    # the reference's data_lib metas: a source time zone to convert from (dropped by its converter), with / without events
    ("trips_case_1.csv", "trips_tz_events.meta.yml", "data_lib/trips_case_1_tz_events.bin"),
    ("trips_case_1.csv", "trips_tz.meta.yml", "data_lib/trips_case_1_tz.bin"),
]


@pytest.mark.parametrize("csv_name,meta_name,ref_bin", PAIRS)
def test_converter_output_is_byte_identical_to_the_reference(tmp_path, csv_name, meta_name, ref_bin):
    ref_bin = os.path.join(G, *ref_bin.split("/"))
    out = str(tmp_path / "out.bin")
    conv = BinaryConverter(out, os.path.join(D, meta_name))
    conv.add_csv(os.path.join(D, csv_name))
    conv.flush()
    conv.close()
    with open(out, "rb") as a, open(ref_bin, "rb") as b:
        got, want = a.read(), b.read()
    assert got == want, (len(got), len(want))
    items, st, et = read_bin(out)
    assert len(items) > 0 and st <= et
    assert int(items["timestamp"].min()) == st and int(items["timestamp"].max()) == et


def test_converter_options_and_edge_cases(tmp_path):
    """several csv files in call order, a fixed start timestamp, values with quotes / decimals, rows that do not parse"""
    meta = tmp_path / "m.yml"
    meta.write_text("entity:\n  timestamp:\n    column: t\n    dtype: i8\n  a:\n    column: a\n    dtype: i\n  b:\n    column: b\n    dtype: f\n"
                    "  missing:\n    column: nope\n    dtype: i2\n  _event: kind\nevents:\n  E1:\n    display_name: e1\n    value_in_csv: 3\n  _default: E1\n")
    c1, c2 = tmp_path / "1.csv", tmp_path / "2.csv"
    c1.write_text('t,a,b\n1970-01-02 00:00:00,"7.9", 1.5 \n100,2,x\n')   # second row: b does not parse -> skipped
    c2.write_text("t,a,b\n50,3,2.25\n")
    out = str(tmp_path / "o.bin")
    with pytest.warns(UserWarning):
        with BinaryConverter(out, str(meta), utc_start_timestamp=10) as conv:
            conv.add_csv(str(c1))
            conv.add_csv(str(c2))
    items, st, et = read_bin(out)
    assert items.dtype.names == ("timestamp", "a", "b", "missing")
    assert items["timestamp"].tolist() == [86400, 50] and items["a"].tolist() == [7, 3]
    assert np.allclose(items["b"], [1.5, 2.25]) and items["missing"].tolist() == [0, 0]
    assert (st, et) == (10, 86400)
