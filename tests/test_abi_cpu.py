"""The C-ABI library builds for sm_90a, loads on a CPU-only box, and exports every symbol include/b200vc.h declares."""
import ctypes
import os
import re

from aicovergen_b200 import _ffi, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    txt = open(os.path.join(ROOT, "include", "b200vc.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(b200vc_[a-z0-9_]+)\s*\(", txt)))


def test_library_builds_and_exports_every_declared_symbol():
    lib_path = build.build()
    assert lib_path.exists()
    lib = ctypes.CDLL(str(lib_path))
    names = _declared()
    assert len(names) >= 25, names
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing


def test_ctypes_struct_mirror_matches_compiled_struct():
    lib = _ffi.lib()          # raises on ABI size mismatch
    assert lib.b200vc_version().startswith(b"b200vc")
    assert lib.b200vc_sizeof_tapgemm_params() == ctypes.sizeof(_ffi.TapGemmParams)


def test_error_reporting_without_gpu():
    """Argument validation happens before any CUDA call, so it is testable here: bad descriptor -> rc<0 + message."""
    lib = _ffi.lib()
    p = _ffi.TapGemmParams()
    rc = lib.b200vc_tapgemm(ctypes.byref(p), 0, None)
    assert rc < 0
    assert b"tapgemm" in lib.b200vc_last_error()


def test_sass_contains_hopper_tensor_and_tma_instructions():
    """wgmma / TMA must survive to SASS in both tensor-core kernels (HGMMA with TF32 and fp16 operands, UTMALDG)."""
    import shutil
    import subprocess

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        import pytest
        pytest.skip("cuobjdump not available")
    for src in ("tapgemm_tc", "tapgemm_ws"):
        obj = build.OUT_DIR / f"{src}.o"
        sass = subprocess.run([cuobjdump, "-sass", str(obj)], capture_output=True, text=True).stdout
        for mnem in ("HGMMA.64x64x8.F32.TF32", "HGMMA.64x64x16.F32", "UTMALDG"):
            assert mnem in sass, (src, mnem)


def test_committed_bench_line_carries_the_contract_keys():
    """The bench line committed under profiles/ (bench.py --gpus 1 --steps 3 --warmup 3 on an H100) has every key the
    JSON contract of bench.py names."""
    import json
    import os

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    b = json.load(open(os.path.join(root, "profiles", "h100_bench.json")))
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline"):
        assert k in b, k
    assert b["config"]["workload"] and b["gpu_launches"] > 0 and b["higher_is_better"] is True and b["scaling"] == "weak"
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(b["e2e"]) and b["e2e"]["h2d_bytes_per_step"] > 0
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(b["roofline"]) and b["roofline"]["bound"] in ("hbm", "tensor")
    assert {"value", "unit", "cores", "kind", "sample"} <= set(b["cpu_baseline"]) and b["cpu_baseline"]["kind"] in ("port", "reference")
    assert {"sm_mhz", "sm_max_mhz", "reasons"} <= set(b["clocks"])
    assert not set(b["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}


def test_plan_recorder_records_instead_of_launching():
    """b200vc_plan_begin .. b200vc_plan_end: entry points called in between are stored (with a copy of their arguments), not
    launched — so this works without a GPU; the plan reports its launch count; misuse returns an error code."""
    from aicovergen_b200 import ops  # noqa: F401  (registers the argtypes)

    lib = _ffi.lib()
    h = ctypes.c_void_p()
    assert lib.b200vc_plan_end() != 0 and b"no plan" in lib.b200vc_last_error()
    assert lib.b200vc_plan_begin(ctypes.byref(h)) == 0 and h.value
    h2 = ctypes.c_void_p()
    assert lib.b200vc_plan_begin(ctypes.byref(h2)) != 0                       # already recording on this thread
    fake = ctypes.c_void_p(0x1000)
    assert lib.b200vc_axpby(fake, None, fake, 16, 1.0, 1.0, None) == 0
    p = _ffi.TapGemmParams()
    p.A, p.Wt, p.out = 0x1000, 0x2000, 0x3000
    p.ntaps, p.BW, p.BH, p.N, p.Kc, p.OW, p.OH, p.OB = 1, 128, 1, 8, 8, 128, 1, 1
    p.a_stride[0] = 1
    assert lib.b200vc_tapgemm(ctypes.byref(p), 0, None) == 0
    assert lib.b200vc_plan_run(h, None) != 0                                   # not while recording
    assert lib.b200vc_plan_end() == 0
    assert lib.b200vc_plan_size(h) == 2 and lib.b200vc_plan_size(None) == -1
    assert lib.b200vc_plan_destroy(h) == 0
