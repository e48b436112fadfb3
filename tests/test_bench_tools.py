"""The benchmark scripts under tools/ share one measurement library (tools/benchlib.py) and never import each other,
so that changing one benchmark cannot silently change what another one measures.  CPU only: the scripts are parsed,
not run."""
import ast
import importlib.util
from pathlib import Path

import pytest

TOOLS = Path(__file__).resolve().parent.parent / "tools"
SCRIPTS = sorted(TOOLS.glob("bench_*.py"))


def imported_modules(path):
    for node in ast.walk(ast.parse(path.read_text(), str(path))):
        if isinstance(node, ast.Import):
            yield from (a.name for a in node.names)
        elif isinstance(node, ast.ImportFrom) and node.module:
            yield node.module


def test_there_are_bench_scripts():
    assert len(SCRIPTS) >= 11


@pytest.mark.parametrize("script", SCRIPTS, ids=lambda p: p.name)
def test_bench_script_imports_no_other_bench_script(script):
    mods = list(imported_modules(script))
    assert "benchlib" in mods
    assert not [m for m in mods if m.split(".")[0].startswith("bench_")]


def test_benchlib_imports_without_a_device_and_rates_windows():
    spec = importlib.util.spec_from_file_location("benchlib", TOOLS / "benchlib.py")
    B = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(B)
    assert B.maps_per_s([30.0, 10.0, 20.0], 256, 5) == 64000.0     # 256 * 5 maps in the median window of 20 ms
    assert B.maps_per_s([3.0], 7, 1) == 2333.33                    # 7 maps in 3 ms, rounded to 2 places
    assert B.default_wave_pairs(450, 375) == 32
