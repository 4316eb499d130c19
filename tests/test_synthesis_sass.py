"""The synthesis recurrence's steady-state block, counted in the SASS of the built library (tools/synthesis_sass.py):
each tap is one IMAD.WIDE.U32 with the accumulator as addend plus one IMAD, with no IADD3 / IADD3.X carry pairs, and a
decoded sample costs at most 25 instructions with 8 taps per lane.  Needs cuobjdump, not a GPU."""
import importlib.util
import pathlib
import shutil

import pytest

ROOT = pathlib.Path(__file__).resolve().parent.parent
LIB = ROOT / "sela_b200" / "libsela_b200.so"


def _tool():
    spec = importlib.util.spec_from_file_location("synthesis_sass", ROOT / "tools" / "synthesis_sass.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.skipif(shutil.which("cuobjdump") is None or not LIB.exists(), reason="needs cuobjdump and the built library")
@pytest.mark.parametrize("kernel", ["k_synthesise_segments", "k_lpc_samples"])
def test_instructions_per_sample(kernel):
    tool = _tool()
    r = tool.analyse(str(LIB), tool.KERNELS[kernel])
    mix = r["opcode_mix_per_sample"]
    assert mix.get("IMAD.WIDE.U32", 0) <= 8 and mix.get("IMAD", 0) <= 8.5, mix
    assert mix.get("IADD3.X", 0) == 0 and mix.get("IMAD.X", 0) == 0, mix
    assert r["per_sample_between_shfl_idx"] <= 25, r
    assert r["whole_run_per_sample"] <= 26, r
