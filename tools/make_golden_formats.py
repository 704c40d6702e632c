"""Write tests/golden/ref_formats.npz and tests/golden/ref_indexed_dataset.{data,idx}: what the original StyleSinger's own
checkpoint loader, IndexedDatasetBuilder and norm_interp_f0 produce on the seeded inputs of tests/test_formats_cpu.py.

    python tools/make_golden_formats.py --src <checkout of the original StyleSinger>

The tests compare stylesinger_b200/formats.py with these stored results, so they need nothing outside the repository.
"""
import argparse
import importlib.util
import json
import os
import shutil
import sys
import tempfile
import types

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
GOLDEN = os.path.join(REPO, "tests", "golden")


def ref_module(src, rel, name, stubs=()):
    for s in stubs:
        sys.modules.setdefault(s, types.ModuleType(s))
    sys.dont_write_bytecode = True  # never write into the original project's tree
    spec = importlib.util.spec_from_file_location(name, os.path.join(src, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", required=True)
    src = ap.parse_args().src
    from tests import test_formats_cpu as T

    out = {}
    # load_ckpt: the newest of two checkpoints, loaded strictly into a fresh module
    ck = ref_module(src, "utils/commons/ckpt_utils.py", "ref_ckpt_utils")
    d = tempfile.mkdtemp()
    try:
        T.write_tiny_checkpoints(d)
        dst = T.Tiny()
        ck.load_ckpt(dst, d, "model", strict=True)
        for k, v in dst.state_dict().items():
            out["ckpt/" + k] = v.numpy()
    finally:
        shutil.rmtree(d)
    # norm_interp_f0 (pitch_norm log, use_uv)
    pu = ref_module(src, "utils/pitch_utils.py", "ref_pitch_utils", stubs=("librosa",))
    for i, f0 in enumerate(T.f0_cases()):
        rf, ru = pu.norm_interp_f0(f0.copy(), {"pitch_norm": "log", "use_uv": True})
        out[f"f0/{i}/in"], out[f"f0/{i}/f0"], out[f"f0/{i}/uv"] = f0, rf.numpy(), ru.numpy()
    out["meta"] = np.array(json.dumps({"source": "original StyleSinger: utils/commons/ckpt_utils.py load_ckpt, "
                                                 "utils/pitch_utils.py norm_interp_f0, utils/commons/indexed_datasets.py"}))
    np.savez_compressed(os.path.join(GOLDEN, "ref_formats.npz"), **out)
    # an IndexedDataset written by the original builder
    ids = ref_module(src, "utils/commons/indexed_datasets.py", "ref_indexed_datasets")
    b = ids.IndexedDatasetBuilder(os.path.join(GOLDEN, "ref_indexed_dataset"))
    for it in T._items():
        b.add_item(it)
    b.finalize()
    print("wrote", GOLDEN)


if __name__ == "__main__":
    main()
