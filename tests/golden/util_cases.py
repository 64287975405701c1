"""Inputs of the host-side input-preparation checks (SUPIR/util.py helpers) and the bit-exact digest their outputs are
recorded with in util_reference.json: shared by tests/golden/make_golden.py (which records the reference's outputs) and
tests/test_util_entry_points.py (which compares this package's outputs with the record)."""
import hashlib

import numpy as np


# cases of the host-side input-preparation helpers (SUPIR/util.py) whose reference outputs are recorded in util_reference.json
PIL2TENSOR_CASES = [(1, 1024, None), (2, 1024, None), (4, 64, None), (1, 1024, 512), (3, 256, 512)]


def pil2tensor_images():
    """24 random images of random sizes, the same stream for the generator and the test."""
    import random
    from PIL import Image
    rng = random.Random(0)
    for _ in range(24):
        w, h = rng.randint(40, 900), rng.randint(40, 900)
        yield w, h, Image.fromarray(np.random.RandomState(w * 1000 + h).randint(0, 255, (h, w, 3), dtype=np.uint8))


def numpy_helper_inputs():
    rng = np.random.RandomState(0)
    hwc3 = [rng.randint(0, 256, shape).astype(np.uint8) for shape in ((17, 23), (17, 23, 1), (17, 23, 3), (17, 23, 4))]
    return hwc3, rng.randint(0, 256, (9, 11, 3)).astype(np.uint8)


def array_digest(a):
    """dtype, shape and sha256 of the raw bytes: a bit-exact record of an array too large to store."""
    a = np.ascontiguousarray(a)
    return {"dtype": str(a.dtype), "shape": list(a.shape), "sha256": hashlib.sha256(a.tobytes()).hexdigest()}
