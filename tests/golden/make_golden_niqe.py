#!/usr/bin/env python
"""Generate tests/golden/niqe_ref.npz from the REAL reference's NIQE: calculate_niqe, niqe, compute_feature and estimate_aggd_param
(Deraining/basicsr/metrics/niqe.py), with reorder_image / to_y_channel (metric_util.py) and bgr2ycbcr (utils/matlab_functions.py),
run with scipy and cv2.  Runs on a development machine with the reference checkout (../reference or $VMB_REFERENCE_DIR); no test
imports it.  It also copies the pristine parameters, unchanged, to tests/golden/niqe_pris_params.npz.

  python tests/golden/make_golden_niqe.py

Nothing is copied from the reference's code: its functions are AST-extracted at run time and executed with `convolve`, `cv2` and `np`
wrapped so that the planes niqe filters and its distparam are recorded.  The inputs are oracle/niqe_ref.case_image's, made from
integer arithmetic only, so a test rebuilds them bit for bit from their seeds.  Stored per case: the input's spec and SHA-256, its
arguments, the score (or the exception's type), the distparam, cv2's half plane as its ulp offset from the float32 2 x 2 mean of the
plane (oracle/niqe_ref.half_plane), the plane at scale 1 (cut to whole blocks) where it is not to_y_channel's or the input's own,
and for two integer cases the scale-1 MSCN map; then scipy's r(gamma) table and the parameter file's SHA-256.
"""
import ast
import hashlib
import math
import os
import shutil
import sys
import types

import cv2
import numpy as np
from scipy.ndimage import convolve
from scipy.special import gamma

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import niqe_ref  # noqa: E402

OUT = mg.OUT
MSCN_CASES = ("u8_crop7", "u16")
PARAMS = f"{mg.REF}/Deraining/basicsr/metrics/niqe_pris_params.npz"


def extract(path, names, ns):
    tree = ast.parse(open(path).read())
    fns = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert {f.name for f in fns} == set(names), (path, names)
    exec(compile(ast.Module(fns, []), path, "exec"), ns)


class Recorder:
    def __init__(self):
        self.conv, self.dist = [], None

    def convolve(self, img, w, mode):
        out = convolve(img, w, mode=mode)
        self.conv.append((img, out))
        return out

    def nanmean(self, a, axis=None):
        self.dist = np.array(a)
        return np.nanmean(a, axis=axis)


def reference(rec):
    npw = types.SimpleNamespace(**{k: getattr(np, k) for k in dir(np) if not k.startswith("__")})
    npw.nanmean = rec.nanmean
    ns = {"np": npw, "cv2": cv2, "math": math, "gamma": gamma, "convolve": rec.convolve}
    b = f"{mg.REF}/Deraining/basicsr"
    extract(f"{b}/utils/matlab_functions.py", ["bgr2ycbcr", "_convert_input_type_range", "_convert_output_type_range"], ns)
    extract(f"{b}/metrics/metric_util.py", ["reorder_image", "to_y_channel"], ns)
    extract(f"{b}/metrics/niqe.py", ["estimate_aggd_param", "compute_feature", "niqe", "calculate_niqe"], ns)
    return ns


def cases():
    """(name, image spec (seed, h, w, c, dtype, flat) for oracle/niqe_ref.case_image, crop_border, input_order, convert_to)"""
    return [("u8_crop0", (1, 196, 290, 3, "uint8", 0), 0, "HWC", "y"),
            ("u8_crop4", (2, 200, 300, 3, "uint8", 0), 4, "HWC", "y"),
            ("u8_crop7", (3, 211, 206, 3, "uint8", 0), 7, "HWC", "y"),
            ("u8_exact", (4, 192, 288, 3, "uint8", 0), 0, "HWC", "y"),
            ("u8_tall", (5, 300, 150, 3, "uint8", 0), 2, "HWC", "y"),
            ("u16", (6, 100, 200, 3, "uint16", 0), 0, "HWC", "y"),
            ("f32_255", (7, 200, 210, 3, "float32", 0), 3, "HWC", "y"),
            ("f64_255", (8, 205, 200, 3, "float64", 0), 0, "HWC", "y"),
            ("u8_chw", (9, 200, 200, 3, "uint8", 0), 1, "CHW", "y"),
            ("f32_hw", (10, 200, 200, 0, "float32", 0), 0, "HW", "y"),
            ("u8_2d_y", (11, 200, 200, 0, "uint8", 0), 0, "HWC", "y"),
            ("u8_gray", (12, 200, 290, 3, "uint8", 0), 5, "HWC", "gray"),
            ("flat_clipped", (13, 200, 300, 3, "uint8", 1), 0, "HWC", "y"),
            ("one_block", (14, 100, 120, 3, "uint8", 0), 0, "HWC", "y"),
            ("small", (15, 80, 120, 3, "uint8", 0), 0, "HWC", "y"),
            ("small_after_crop", (16, 100, 130, 3, "uint8", 0), 4, "HWC", "y")]


def image(spec, order):
    """the case's input as the reference receives it (CHW: transposed)"""
    seed, h, w, c, dtype, flat = spec
    img = niqe_ref.case_image(seed, h, w, c, dtype, bool(flat))
    return np.ascontiguousarray(img.transpose(2, 0, 1)) if order == "CHW" else img


def main():
    data, names = {}, []
    here = os.getcwd()
    for name, spec, crop, order, conv in cases():
        rec = Recorder()
        ref = reference(rec)
        names.append(name)
        img = image(spec, order)
        data[f"{name}/spec"] = np.array([str(v) for v in spec])
        data[f"{name}/img_sha256"] = np.array(hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest())
        data[f"{name}/meta"] = np.array([str(crop), order, conv])
        os.chdir(f"{mg.REF}/Deraining")  # calculate_niqe loads basicsr/metrics/niqe_pris_params.npz from the working directory
        try:
            with np.errstate(all="ignore"):
                data[f"{name}/score"] = np.asarray(ref["calculate_niqe"](img, crop, input_order=order, convert_to=conv))
            data[f"{name}/raises"] = np.array("")
        except np.linalg.LinAlgError:
            data[f"{name}/raises"] = np.array("LinAlgError")
        except cv2.error:
            data[f"{name}/raises"] = np.array("cv2.error")
        finally:
            os.chdir(here)
        if rec.dist is not None:
            data[f"{name}/features"] = rec.dist
        if len(rec.conv) == 4:
            (plane, mu), (_, c2), (half, _), _ = rec.conv
            # cv2's half plane, exactly, as its ulp offset from the float32 2 x 2 mean (the library's half plane) of the plane
            ulp = half.view(np.int32).astype(np.int64) - niqe_ref.half_plane(plane).view(np.int32)
            assert np.abs(ulp).max() <= 127
            data[f"{name}/half_ulp"] = ulp.astype(np.int8)
            if conv == "gray":  # the Y and 'HW' planes are recomputed bit for bit from the input (oracle/metrics_ref.py)
                data[f"{name}/plane"] = plane
            if name in MSCN_CASES:  # the reference's MSCN expression, on its own filter outputs
                data[f"{name}/mscn"] = (plane - mu) / (np.sqrt(np.abs(c2 - np.square(mu))) + 1)
        print(name, data[f"{name}/raises"], data.get(f"{name}/score"))
    g = np.arange(0.2, 10.001, 0.001)
    data["r_gam"] = np.square(gamma(np.reciprocal(g) * 2)) / (gamma(np.reciprocal(g)) * gamma(np.reciprocal(g) * 3))
    data["params_sha256"] = np.array(hashlib.sha256(open(PARAMS, "rb").read()).hexdigest())
    data["cases"] = np.array(names)
    shutil.copyfile(PARAMS, os.path.join(OUT, "niqe_pris_params.npz"))
    path = os.path.join(OUT, "niqe_ref.npz")
    np.savez_compressed(path, **data)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
