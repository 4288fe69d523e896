"""Writes tests/golden/fmi_writer_golden.json: the SHA-256 of the .fmi file the reference's own FMIndex::save
(compiled into oracle/_ref by `make -C oracle ref`) writes for each text of
tests/test_host_logic.py::test_sdsl_format_writer_round_trip_and_reference_bytes.

    python tests/golden/make_fmi_writer_golden.py
"""
import hashlib
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))


def main():
    from oracle.fm_oracle import RefFM, ref_available
    from test_host_logic import _fmi_writer_texts
    assert ref_available(), "oracle/_ref not built"
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for name, text in _fmi_writer_texts().items():
            p = os.path.join(d, "ref.fmi")
            RefFM(np.asarray(text, dtype=np.uint64)).save(p)
            with open(p, "rb") as f:
                out[name] = hashlib.sha256(f.read()).hexdigest()
    with open(os.path.join(HERE, "fmi_writer_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
