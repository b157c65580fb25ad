"""The boundary is a C ABI: include/lcd_b200.h must compile as plain C99, every declared entry point must link from a C program,
and without a CUDA device lcd_create must fail loudly (NULL + a message) instead of falling back to anything."""
import shutil
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from rtabmap_b200 import capi  # noqa: E402


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no C compiler")
def test_header_is_c99_and_every_symbol_links(tmp_path):
    lib = capi.library_path()
    if not lib.exists():
        from rtabmap_b200 import build
        build.build()
    names = sorted(capi.SIGNATURES)
    src = ['#include "lcd_b200.h"', "#include <stdio.h>", "#include <string.h>", "typedef void (*fn_t)(void);", "int main(void)", "{",
           "\tfn_t fns[] = {" + ", ".join(f"(fn_t){n}" for n in names) + "};",
           "\tunsigned i, n = 0;",
           "\tfor (i = 0; i < sizeof(fns) / sizeof(fns[0]); ++i) n += fns[i] != 0;",
           "\tlcd_config cfg;", "\tmemset(&cfg, 0, sizeof(cfg));", "\tcfg.desc_type = LCD_DESC_U8;", "\tcfg.desc_dim = 32;",
           "\tlcd_engine * e = lcd_create(&cfg);",
           '\tprintf("%u %d %s %d %s\\n", n, lcd_abi_version(), lcd_build_arch(), e != 0, e ? "" : lcd_last_error(0));',
           "\tif (e) lcd_destroy(e);", "\treturn 0;", "}"]
    c = tmp_path / "abi.c"
    c.write_text("\n".join(src) + "\n")
    exe = tmp_path / "abi"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(c), "-L", str(lib.parent), "-llcd_b200",
                        f"-Wl,-rpath,{lib.parent}", "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    n, abi, arch, created, *msg = out.stdout.split(" ", 4)
    assert int(n) == len(names) and int(abi) >= 1 and arch == "sm_90a"
    import torch
    if not torch.cuda.is_available():
        # no device here: creation must fail with an explanation, never hand back a CPU engine
        assert created == "0" and "CUDA" in " ".join(msg)
