"""What the unmodified reference printed for the seeded inputs of the tests that compare against it
(tests/golden/ref_live.json, written by tests/golden/make_golden_ref_live.py): sha256 and length of each output."""
import hashlib
import json
import os

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_live.json")


def load(section):
    with open(PATH) as f:
        return json.load(f)[section]


def matches(data, want) -> bool:
    if isinstance(data, str):
        data = data.encode()
    return len(data) == want["bytes"] and hashlib.sha256(data).hexdigest() == want["sha256"]
