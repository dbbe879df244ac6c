"""The DEFLATE entry points from a plain-C client (strict C11), without a device."""
import os
import shutil
import subprocess

import pytest

from conftest import ROOT


def test_deflate_client_compiles_links_and_runs(lib, tmp_path):
    if not shutil.which("gcc"):
        pytest.skip("no C compiler")
    exe = str(tmp_path / "deflate_client")
    pkg = os.path.join(ROOT, "pixo_b200")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "c", "deflate_client.c"), "-o", exe, "-L", pkg, "-lpixo_b200",
                    f"-Wl,-rpath,{pkg}"], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "deflate_client ok" in out.stdout, (out.returncode, out.stdout, out.stderr)


def test_new_symbols_are_bound(lib):
    from pixo_b200 import _lib
    for name in ("pixo_b200_deflate_zlib", "pixo_b200_deflate_zlib_on_device"):
        assert name in _lib.SYMBOLS and hasattr(lib, name)
    assert _lib.ERR_INVALID_COMPRESSION_LEVEL == 14
