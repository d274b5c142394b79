"""The GEMM-worker entry point (PB2_LINK_GEMM_BODY_ENTRY, pb2_linked_gemm_body), host side.

  - the flag's value, from C and from Python;
  - the link calls: the flag needs a nonzero GEMM-worker mask (and so PB2_LINK_GEMM_WINDOWS); a refusal records nothing;
  - the device ABI header states the entry point and its register budget;
  - the fixture (tests/cuda/gemm_entry_bodies.cu) links offline with the engine's entry build of the GEMM kernels within
    both budgets, and its DGEMM keeps every DMMA clear of local memory; an image without the entry point, or the
    fixture compiled without -maxrregcount, does not link.
The GPU side is tests/test_gemm_body_entry_gpu.py."""
import os
import re
import subprocess

import pytest

from parsec_b200 import _lib as L
from parsec_b200 import runtime as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
BUILD = os.path.join(ROOT, "build")
FIXTURE = os.path.join(ROOT, "tests", "cuda", "gemm_entry_bodies.cu")
ENTRY = 0x2
GEMM_BODIES = 0x03


def tool(name):
    return os.path.join(CUDA, "bin", name)


# ----------------------------------------------------------------------------------------------------------------------
# the flag and the link calls
# ----------------------------------------------------------------------------------------------------------------------
def test_flag_value(tmp_path):
    assert L.LINK_GEMM_BODY_ENTRY == ENTRY
    src = tmp_path / "flag.c"
    src.write_text('#include <stdio.h>\n#include <stdint.h>\n#include <stddef.h>\n#include "pb2_engine.h"\n'
                   'int main(void) { printf("%u", (unsigned)PB2_LINK_GEMM_BODY_ENTRY); return 0; }\n')
    exe = tmp_path / "flag"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe),
                           str(src)])
    assert subprocess.check_output([str(exe)]) == b"2"


@pytest.fixture(scope="module")
def args_error(tmp_path_factory):
    """why(flags, sliceable): the message of link_args_error, the check every link call makes, or "" for none."""
    d = tmp_path_factory.mktemp("link_args")
    src = d / "why.cpp"
    src.write_text('#include <cstdio>\n#include <cstdlib>\n#include "pb2_engine_priv.hpp"\n'
                   'int main(int, char** v) { const char* w = link_args_error("x", 1, PB2_IMAGE_PTX, '
                   '(uint32_t)strtoul(v[2], 0, 0), 0, (uint32_t)strtoul(v[1], 0, 0)); printf("%s", w ? w : ""); }\n')
    exe = d / "why"
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(CUDA, "include"), "-I" + os.path.join(ROOT, "parsec_b200", "csrc"),
                    str(src), "-o", str(exe)], check=True)
    return lambda flags, sliceable=0: subprocess.check_output([str(exe), hex(flags), hex(sliceable)], text=True)


def link(flags, sliceable=0):
    """rc of a dry-run pb2_device_link_bodies_ex with these flags; then that of a valid entry link, and of a second."""
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        dev = ctx.devices[0]
        rc = ctx.l.pb2_device_link_bodies_ex(dev, b"x", 1, L.IMAGE_PTX, sliceable, 0, flags)
        valid = L.LINK_GEMM_WINDOWS | L.LINK_GEMM_BODY_ENTRY | L.LINK_GEMM_BODIES(GEMM_BODIES)
        after = ctx.l.pb2_device_link_bodies_ex(dev, b"x", 1, L.IMAGE_PTX, 0, 0, valid)
        second = ctx.l.pb2_device_link_bodies_ex(dev, b"x", 1, L.IMAGE_PTX, 0, 0, 0)
    return rc, after, second


@pytest.mark.parametrize("flags", [ENTRY, ENTRY | L.LINK_GEMM_WINDOWS,
                                   ENTRY | L.LINK_GEMM_WINDOWS | L.LINK_READERS(0x04) | L.LINK_READER_GROUPS(0x04)],
                         ids=["alone", "gemm_windows", "readers"])
def test_refused_without_a_gemm_worker_mask(args_error, flags):
    rc, after, second = link(flags, sliceable=0x04)
    assert rc == L.PB2_ERR_BAD_PARAM
    why = args_error(flags, 0x04)
    assert "PB2_LINK_GEMM_BODY_ENTRY without a PB2_LINK_GEMM_BODIES mask" in why and "unknown bit" not in why
    # nothing was recorded: a valid link still succeeds, and then a second one is refused as one
    assert after == 0 and second == L.PB2_ERR_EXISTS


def test_refused_without_gemm_windows(args_error):
    flags = ENTRY | L.LINK_GEMM_BODIES(GEMM_BODIES)
    rc, after, second = link(flags)
    assert rc == L.PB2_ERR_BAD_PARAM and "without PB2_LINK_GEMM_WINDOWS" in args_error(flags)
    assert after == 0 and second == L.PB2_ERR_EXISTS


@pytest.mark.parametrize("flags", [0x4, 0x80, ENTRY | 0x4], ids=["bit2", "bit7", "entry_and_bit2"])
def test_other_low_bits_are_still_unknown(args_error, flags):
    flags |= L.LINK_GEMM_WINDOWS | L.LINK_GEMM_BODIES(GEMM_BODIES)
    rc, after, second = link(flags)
    why = args_error(flags)
    assert rc == L.PB2_ERR_BAD_PARAM and "unknown bit" in why and "PB2_LINK_GEMM_BODY_ENTRY" in why
    assert after == 0 and second == L.PB2_ERR_EXISTS


@pytest.mark.parametrize("kw", [dict(gemm_bodies=0x01), dict(gemm_bodies=0xFF),
                                dict(gemm_bodies=0x01, sliceable=0x06, readers=0x04, reader_groups=0x04)],
                         ids=["one", "all_eight", "with_reader_groups"])
def test_accepted_with_a_mask(args_error, kw):
    flags = (L.LINK_GEMM_WINDOWS | ENTRY | L.LINK_GEMM_BODIES(kw["gemm_bodies"]) | L.LINK_READERS(kw.get("readers", 0))
             | L.LINK_READER_GROUPS(kw.get("reader_groups", 0)))
    assert args_error(flags, kw.get("sliceable", 0)) == ""
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        dev = ctx.devices[0]
        ctx.link_bodies(dev, b"ptx", L.IMAGE_PTX, gemm_windows=True, gemm_body_entry=True, **kw)
        assert ctx.l.pb2_device_link_bodies_ex(dev, b"x", 1, L.IMAGE_PTX, 0, 0, 0) == L.PB2_ERR_EXISTS


def test_python_refusal_raises():
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        with pytest.raises(L.Pb2Error) as ex:
            ctx.link_bodies(ctx.devices[0], b"ptx", L.IMAGE_PTX, gemm_windows=True, gemm_body_entry=True)
        assert ex.value.rc == L.PB2_ERR_BAD_PARAM


def test_engine_link_refuses_a_null_engine():
    lib = L.load()
    flags = L.LINK_GEMM_WINDOWS | L.LINK_GEMM_BODY_ENTRY | L.LINK_GEMM_BODIES(GEMM_BODIES)
    assert lib.pb2_engine_link_bodies_ex(None, b"x", 1, L.IMAGE_CUBIN, 0, 0, flags) == L.PB2_ERR_BAD_PARAM


# ----------------------------------------------------------------------------------------------------------------------
# the device ABI header
# ----------------------------------------------------------------------------------------------------------------------
def test_header_states_the_entry_point_and_its_budget(tmp_path):
    src = tmp_path / "regs.c"
    src.write_text('#include <stdio.h>\n#include "pb2_device_body.h"\n'
                   'int main(void) { printf("%d\\n", PB2_GEMM_BODY_MAX_REGS); return 0; }\n')
    exe = tmp_path / "regs"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                   check=True)
    assert int(subprocess.check_output([str(exe)], text=True)) == 168
    hdr = open(os.path.join(ROOT, "include", "pb2_device_body.h")).read()
    assert re.search(r'extern "C" __device__ unsigned long long pb2_linked_gemm_body\(int body, const pb2_body_args_t\* a,'
                     r'\s+unsigned int\* scratch\);', hdr)
    # the GEMM window kernels' budget is the header's: __launch_bounds__(384, 1) gives 168 registers a thread
    gemm = open(os.path.join(ROOT, "parsec_b200", "csrc", "pb2_gemm.cuh")).read()
    assert "__launch_bounds__(gemm::kThreads, 1)" in gemm and "constexpr int kThreads = 384;" in gemm


# ----------------------------------------------------------------------------------------------------------------------
# the fixture, linked offline
# ----------------------------------------------------------------------------------------------------------------------
def built(*names):
    paths = [os.path.join(BUILD, n) if n.endswith(".cubin") and n.startswith("pb2_") else os.path.join(ROOT, "tests", "cuda", n)
             for n in names]
    assert all(os.path.exists(p) for p in paths), "build() makes the engine cubins and the fixtures"
    return paths


def nvlink(tmp_path, inputs):
    out = tmp_path / "linked.cubin"
    p = subprocess.run([tool("nvlink"), "-arch=sm_90a", "-o", str(out), *inputs], capture_output=True, text=True)
    return p, out


def resources(cubin):
    res = subprocess.check_output([tool("cuobjdump"), "-res-usage", str(cubin)], text=True)
    gemm = re.findall(r"Function _ZN3pb223pb2_engine_gemm2_kernelI\w+:\s*\n\s*REG:(\d+) STACK:\d+ SHARED:(\d+)", res)
    hbm = re.findall(r"Function _ZN3pb221pb2_engine_hbm_kernelI\w+:\s*\n\s*REG:(\d+)", res)
    return [(int(r), int(s)) for r, s in gemm], [int(r) for r in hbm]


@pytest.mark.parametrize("gemm_cubin,bodies", [("pb2_engine_linked_gemm_entry.cubin", "gemm_entry_bodies.cubin"),
                                               ("pb2_engine_linked_gemm_entry_groups.cubin", "gemm_entry_group_bodies.cubin")],
                         ids=["entry", "entry_groups"])
def test_fixture_links_within_both_budgets(tmp_path, gemm_cubin, bodies):
    hbm_cubin = "pb2_engine_linked_groups.cubin" if "groups" in gemm_cubin else "pb2_engine_linked.cubin"
    p, out = nvlink(tmp_path, built(hbm_cubin, gemm_cubin, bodies))
    assert p.returncode == 0, p.stderr
    assert "C7509" not in p.stdout + p.stderr
    gemm, hbm = resources(out)
    assert len(gemm) == 4 and len(hbm) == 4
    assert all(r <= 168 and s + 196608 + 1024 <= 227 * 1024 for r, s in gemm), gemm
    assert all(r == 80 for r in hbm), hbm


def test_dgemm_keeps_local_memory_out_of_its_dmma_loop():
    """ptxas reports spill stores for pb2_linked_gemm_body: the call ABI's saves of callee-saved registers.  None of
    them, and no other local access, lies between the first and the last DMMA."""
    sass = subprocess.check_output([tool("cuobjdump"), "-sass", "-fun", "pb2_linked_gemm_body",
                                    *built("gemm_entry_bodies.cubin")], text=True).splitlines()
    dmma = [i for i, l in enumerate(sass) if "DMMA.8x8x4" in l or "DMMA.16x8x8" in l]
    assert len(dmma) >= 16, "the DGEMM body runs on the FP64 tensor cores"
    local = [l.strip() for l in sass[dmma[0]:dmma[-1]] if re.search(r"\b(LDL|STL)\b", l)]
    assert not local, local[:8]
    log = open(os.path.join(ROOT, "tests", "cuda", "gemm_entry_bodies.log")).read()
    body = re.search(r"Function properties for pb2_linked_body\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores", log)
    assert body and body.group(2) == "0", log


def test_entry_kernels_need_the_symbol(tmp_path):
    """The entry build of the GEMM kernels with an image that defines pb2_linked_body alone: undefined reference."""
    p, _ = nvlink(tmp_path, built("pb2_engine_linked.cubin", "pb2_engine_linked_gemm_entry.cubin", "gemm_worker_bodies.cubin"))
    assert p.returncode != 0 and "pb2_linked_gemm_body" in p.stderr and "ndefined" in p.stderr, p.stderr
    # the plain build never names it: the same image links
    p, _ = nvlink(tmp_path, built("pb2_engine_linked.cubin", "pb2_engine_linked_gemm.cubin", "gemm_worker_bodies.cubin"))
    assert p.returncode == 0, p.stderr


def test_fixture_without_the_register_cap_is_refused(tmp_path):
    """Compiled without -maxrregcount, the DGEMM needs more than the GEMM kernels' 168 registers, which nvlink refuses."""
    uncapped = tmp_path / "uncapped.cubin"
    subprocess.check_call([tool("nvcc"), "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-rdc=true",
                           "-cubin", "-I" + os.path.join(ROOT, "include"), "-o", str(uncapped), FIXTURE])
    p, _ = nvlink(tmp_path, built("pb2_engine_linked.cubin", "pb2_engine_linked_gemm_entry.cubin") + [str(uncapped)])
    assert p.returncode != 0, p.stdout
    assert re.search(r"max regcount of 168 calls function 'pb2_linked_gemm_body' with regcount of \d+", p.stderr), p.stderr
