"""The hot-key collectors' host logic (incubator_pegasus_b200/host/hotkey.h): the golden find_outlier_index cases of the
reference's unit test (tests/golden/hotkey_outliers.json) and its state-transition and fine-collector sequences, run as a C++
unit test (tests/cpp/test_hotkey.cpp) under ThreadSanitizer and AddressSanitizer; and the Python model the GPU tests compare
the library with (tests/hotkey_model.py) against the same cases."""
import json
import os
import shutil
import subprocess

import pytest

import hotkey_model as hm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "hotkey_outliers.json")


def cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("sanitizer", ["thread", "address,undefined"])
def test_hotkey_host_collector(tmp_path, sanitizer):
    cxx = shutil.which("g++")
    assert cxx, "g++ is part of this image"
    txt = tmp_path / "cases.txt"
    txt.write_text("".join("%d %d %d %d %s\n" % (c["threshold"], int(c["found"]), c["index"], len(c["values"]),
                                                  " ".join(str(v) for v in c["values"])) for c in cases()))
    exe = str(tmp_path / "test_hotkey")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-g", "-pthread", f"-fsanitize={sanitizer}",
                           os.path.join(ROOT, "tests", "cpp", "test_hotkey.cpp"), "-o", exe])
    out = subprocess.run([exe, str(txt)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr
    assert "outlier cases: %d" % len(cases()) in out.stdout
    assert "WARNING: ThreadSanitizer" not in out.stderr and "runtime error" not in out.stderr, out.stderr


@pytest.mark.parametrize("case", cases(), ids=lambda c: c["source"])
def test_model_outliers(case):
    assert hm.find_outlier_index(case["values"], case["threshold"]) == (case["found"], case["index"])


def test_model_state_machine():
    c = hm.Collector()
    assert c.control(hm.QUERY, 0) == hm.BUSY and c.control(hm.START, 0) == hm.OK and c.control(hm.START, 1) == hm.BUSY
    for _ in range(200):
        c.capture_raw_key(b"\x00\x03hotsort")
    for i in range(100):
        c.capture_raw_key(b"\x00\x04k%03d" % i)
    c.analyse(10)
    assert c.state == hm.FINE and c.target == hm.bucket(b"hot", 37)
    for _ in range(50):
        c.capture_hash_key(b"hot", 2)
    c.analyse(20)
    assert c.state == hm.FINISHED and c.result == b"hot" and c.control(hm.START, 21) == hm.BUSY
    assert c.control(hm.STOP, 22) == hm.OK and c.state == hm.STOPPED and c.result == b""
    c.control(hm.START, 100)
    c.analyse(249)
    assert c.state == hm.COARSE
    c.analyse(250)
    assert c.state == hm.STOPPED
