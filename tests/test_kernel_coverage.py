"""Every entry point of include/masr_b200.h is called by name in some test, or listed below with the reason it is not.

A kernel added to the header without a test that names it fails here, on the CPU suite."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "masr_b200.h")

# entry point -> why no test names it as a string
COVERED_INDIRECTLY = {
    "masr_abi_version": "called as a ctypes attribute in test_abi.py::test_abi_version_and_error_string",
    "masr_lm_load_arpa": "through CharLM in test_lm.py and test_gpu_lm.py, including every rejected file",
    "masr_lm_info": "through CharLM in test_lm.py and test_gpu_lm.py",
    "masr_lm_export": "through CharLM in test_lm.py and test_gpu_lm.py",
    "masr_lm_free": "through CharLM in test_lm.py and test_gpu_lm.py",
    "masr_lm_score_f32": "through CharLM.score in test_gpu_lm.py, bit for bit against oracle/lm.py",
}


def header_entry_points():
    with open(HEADER, encoding="utf-8") as f:
        text = f.read()
    return re.findall(r"^\s*(?:const\s+char\s*\*|int)\s+(masr_\w+)\s*\(", text, re.M)


def test_header_is_parsed():
    names = header_entry_points()
    assert len(names) == len(set(names)) and len(names) >= 50
    assert "masr_lstm_step_f32" in names and "masr_last_error" in names


def test_every_entry_point_is_tested():
    texts = []
    for path in sorted(glob.glob(os.path.join(ROOT, "tests", "*.py"))):
        if os.path.basename(path) != os.path.basename(__file__):
            with open(path, encoding="utf-8") as f:
                texts.append(f.read())
    corpus = "\n".join(texts)
    names = header_entry_points()
    untested = [n for n in names if n not in COVERED_INDIRECTLY and not re.search(r"[\"']" + n + r"[\"']", corpus)]
    assert not untested, f"entry points no test calls by name (add a test, or an entry with a reason): {untested}"
    stale = sorted(set(COVERED_INDIRECTLY) - set(names))
    assert not stale, f"allowlisted names that are not in the header: {stale}"
    assert all(reason.strip() for reason in COVERED_INDIRECTLY.values())
