"""Rebuild the mini-dataset of tests/golden/data_pipeline.npz (oracle/make_pipeline_golden.py) from the bytes it stores."""
import json
import os

import numpy as np

from tests._util import ROOT

GOLD = os.path.join(ROOT, "tests", "golden", "data_pipeline.npz")


def load_golden():
    with np.load(GOLD) as d:
        return {k: d[k] for k in d.files}


def write_inputs(g, base):
    for k, v in g.items():
        if k.startswith("file:"):
            p = os.path.join(base, k[len("file:"):])
            os.makedirs(os.path.dirname(p), exist_ok=True)
            with open(p, "wb") as f:
                f.write(v.tobytes())
    return base


def data_definition(g):
    return json.loads(g["data_definition"].tobytes().decode())


def conf_for(base, processed="processed"):
    with open(os.path.join(ROOT, "ubisoft-laforge-zeroeggs_b200", "data", "data_pipeline_conf_v1.json")) as f:
        conf = json.load(f)
    conf.update(base_path=str(base), processed_data_path=processed, info_filename="info.csv")
    return conf
