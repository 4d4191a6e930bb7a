"""Write tests/golden/validation_windows.npz: what the reference's SGDataset (ZEGGS/dataset.py) returns on the synthetic fixture of
tests/test_validation_cpu.py -- its window enumeration over the validation ranges, the rows of the style example of every
validation tile and the sample clips of get_sample / get_example.  Needs the reference tree (oracle/ref_shim.py)."""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.test_validation_cpu import reference_values  # noqa: E402

if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as d:
        out = reference_values(d)
    path = os.path.join(ROOT, "tests", "golden", "validation_windows.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, sum(v.nbytes for v in out.values()), "bytes")
