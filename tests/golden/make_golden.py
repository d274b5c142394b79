#!/usr/bin/env python
"""Generates tests/golden/reference_runtime_cpu.json: the answers of the UNMODIFIED reference runtime (oracle/_ref/parsec,
built from /root/reference by oracle/build_ref_runtime.sh) running the test applications of tests/parsec with their CPU
incarnations only -- no device module of ours is loaded.  Run where oracle/_ref/bin exists (this container); the GPU tests
compare what the b200 component produces for the same command lines against these records (tests/test_golden.py).
Only the deterministic fields are kept: counts, error totals and the FNV-1a checksum of the final host data (bit-exact
comparison of what the DAG computed), not timings."""
import json
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
BIN = os.path.join(ROOT, "oracle", "_ref", "bin")
CASES = {
    # name: (app, args for the CPU run of the reference, args for the GPU run through the component, fields that must agree)
    "ex05_K128": ("ex05_b200", ["-K", 128, "-t", 65536, "-c", 4, "-w"], ["checksum", "tasks", "errors", "K", "NB", "F", "tile_bytes"]),
    "ex05_K512_r2": ("ex05_b200", ["-K", 512, "-t", 65536, "-c", 8, "-r", 2], ["tasks", "errors", "K", "NB", "F", "tile_bytes", "repeats"]),
    "ex02_N999": ("ex02_b200", ["-N", 999, "-c", 2, "-r", 3], ["checksum", "tasks", "errors", "NB", "repeats"]),
    "stage_4x3": ("stage_b200", ["-c", 4], ["checksum", "tiles", "check_errors", "host_errors"]),
    "dtd_M16": ("dtd_b200", ["-M", 16, "-n", 4096, "-N", 8, "-c", 4], ["checksums", "tiles", "nb", "hops", "errors", "total_errors"]),
    "batch_M96": ("batch_b200", ["-M", 96, "-c", 4], ["checksum", "tiles", "errors"]),
}
CPU_FLAG = {"ex05_b200": ["-m", "cpu"], "ex02_b200": ["-m", "cpu"], "stage_b200": ["-m", "cpu"], "dtd_b200": ["-C"], "batch_b200": ["-m", "cpu"]}


def run(app, args):
    env = dict(os.environ, PARSEC_MCA_device_cuda_enabled="0")
    for k in ("PARSEC_MCA_device_b200_enabled", "PARSEC_MCA_device_b200_dry_run"):
        env.pop(k, None)
    p = subprocess.run([os.path.join(BIN, app)] + [str(a) for a in args], env=env, cwd="/tmp", capture_output=True, text=True, timeout=300)
    line = [l for l in p.stdout.splitlines() if l.startswith("{")][-1]
    return p.returncode, json.loads(line)


def record_reference_pieces():
    """tests/golden/reference_pieces.json.gz: the answers of the reference pieces of oracle/_ref (zone_malloc.c, data.c,
    the 2D block-cyclic collection, device selection) to the call sequences of tests/test_oracle.py, which replays them
    where oracle/_ref is not built."""
    import gzip
    import sys
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_oracle as T
    assert T.HAVE_REF_ZONE and T.HAVE_REF_DATA and T.HAVE_REF_TWODBC and T.HAVE_REF_SELECT, "build oracle/_ref first"
    T.test_zone_oracle_equals_reference_build()
    T.test_coherency_oracle_equals_reference_build()
    T.test_twodbc_oracle_and_product_equal_reference_build()
    T.test_select_oracle_equals_reference_build()
    with gzip.GzipFile(T.GOLDEN_PIECES, "wb", mtime=0) as f:
        f.write(json.dumps(T.RECORDED, separators=(",", ":")).encode())
    print("wrote", T.GOLDEN_PIECES)


if __name__ == "__main__":
    record_reference_pieces()
    out = {}
    for name, (app, args, fields) in CASES.items():
        rc, d = run(app, CPU_FLAG[app] + args)
        assert rc == 0, (name, rc, d)
        out[name] = {"app": app, "args": [str(a) for a in args], "rc": rc, "fields": {f: d[f] for f in fields}}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_runtime_cpu.json")
    json.dump(out, open(path, "w"), indent=1, sort_keys=True)
    print("wrote", path)
