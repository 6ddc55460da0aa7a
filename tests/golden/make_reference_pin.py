#!/usr/bin/env python
"""Record the reference's outputs that a reference-pin test module compares the oracle against: by default
tests/golden/reference_pin_v1.npz for tests/test_reference_pin.py.  Needs a GPU and the reference libraries
oracle/build_ref.py builds into oracle/_ref/.  It runs every test of the module against the live reference (so the
comparisons are checked while recording) and stores each output the reference returns through ref_lib.PinnedRef.

  python tests/golden/make_reference_pin.py [OUT.npz]                  (tests/test_reference_pin.py)
  python tests/golden/make_reference_pin.py MODULE OUT.npz             (e.g. test_reference_pin_cases)

The module's tests take the `reference` fixture: reference(tag, L, res, nofma) -> a PinnedRef.  A module that sets
PACKED = True is stored in ref_lib.pack's form (a few arrays, not two per call) and reads it with ref_lib.Packed.
"""
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import importlib  # noqa: E402

import ref_lib  # noqa: E402


def main():
    if len(sys.argv) > 2:
        module, out = sys.argv[1], sys.argv[2]
    else:
        module = "test_reference_pin"
        out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "reference_pin_v1.npz")
    pin = importlib.import_module(module.removesuffix(".py").replace("tests/", "").replace("/", "."))
    import torch
    assert torch.cuda.is_available(), "the reference runs on a GPU"
    assert ref_lib.available(True) and ref_lib.available(False), "oracle/_ref is not built (oracle/build_ref.py)"
    store = {}

    def live(tag, L, res, nofma):
        return ref_lib.PinnedRef(store, tag, live=ref_lib.RefMap(L, res, nofma=nofma))

    tests = [getattr(pin, n) for n in dir(pin) if n.startswith("test_")]
    for t in tests:
        t0 = time.perf_counter()
        t(live)
        print(f"recorded {t.__name__} in {time.perf_counter() - t0:.1f} s", file=sys.stderr)
    if getattr(pin, "PACKED", False):
        store = ref_lib.pack(store)
    store["generated_by"] = np.array("reference gpu_process.cu on " + torch.cuda.get_device_name(0))
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **store)
    print("wrote", out, os.path.getsize(out), "bytes;", str(store["generated_by"]), file=sys.stderr)


if __name__ == "__main__":
    main()
