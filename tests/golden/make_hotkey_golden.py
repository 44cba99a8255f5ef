#!/usr/bin/env python
"""Regenerates hotkey_outliers.json: the find_outlier_index cases of the reference's
src/server/test/hotkey_collector_test.cpp:83-104 (inputs, threshold, the expected found flag and hot index), plus the two
standard_deviation == 0 shapes its comment names (hotkey_collector.cpp:112-119) and an all-zero input, whose answers are
read off the reference's code: the largest value is hot when it lies above the average of the others, and hot_index keeps
the first largest value when it does not (that branch does not reset it); with no value above zero it stays -1.
tests/test_hotkey_host.py checks the library's host collector and the Python model against every case."""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))

CASES = [
    # hotkey_collector_test.cpp:89-104 (threshold 3)
    {"values": [1, 2, 3], "threshold": 3, "found": False, "index": -1, "source": "hotkey_collector_test.cpp:89-91"},
    {"values": [1, 2, 100000], "threshold": 3, "found": True, "index": 2, "source": "hotkey_collector_test.cpp:93-95"},
    {"values": [1, 10000, 2, 3, 4, 10000000, 6], "threshold": 3, "found": True, "index": 5, "source": "hotkey_collector_test.cpp:97-99"},
    {"values": list(range(1, 16)), "threshold": 3, "found": False, "index": -1, "source": "hotkey_collector_test.cpp:101-104"},
    # hotkey_collector.cpp:112-119: the values other than the largest are all equal
    {"values": [1, 1, 300, 1], "threshold": 3, "found": True, "index": 2, "source": "hotkey_collector.cpp:113 (case 1)"},
    {"values": [1, 1, 1, 1], "threshold": 3, "found": False, "index": 0, "source": "hotkey_collector.cpp:114 (case 2)"},
    {"values": [0, 0, 0], "threshold": 7, "found": False, "index": -1, "source": "hotkey_collector.cpp:97-99 (nothing above 0)"},
]


def main():
    with open(os.path.join(HERE, "hotkey_outliers.json"), "w") as f:
        json.dump({"source": "reference src/server/test/hotkey_collector_test.cpp find_outlier_index_test", "cases": CASES}, f, indent=1)
    print("cases:", len(CASES))


if __name__ == "__main__":
    main()
