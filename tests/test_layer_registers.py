"""Register budget of the recurrent kernel (csrc/lstm_layer.cu), read from the library build: the `-Xptxas -v` log that
csrc/Makefile writes for lstm_layer.cu and the SASS of its object file.

Warpgroup 0 (producers, counter watcher) gives its registers to the two consumer warpgroups with setmaxnreg, so that
the consumers can hold an item's epilogue inputs (c_{t-1}, fp16 Gx, the pooled running max) in registers while its
last MMAs run. ptxas drops setmaxnreg without an error (only a C7507 note) when a kernel makes an out-of-line call,
and the consumers then spill; these tests pin that the budgets took effect in every instantiation.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "code_intelligence_b200", "csrc", "build")

# spill stores (bytes) allowed per kernel family, as recorded in DESIGN.md §6 ("Registers moved to the consumers"):
# the fused last layer spills in its epilogue only (never inside the K loop, checked below)
SPILL_LIMITS = {
    "lstm_layer_kernel": 0,
    "lstm_layer_mc_kernel": 0,
    "lstm_layer_fused_kernel<false": 212,
    "lstm_layer_fused_kernel<true": 568,
}


def _demangled_family(mangled):
    m = re.search(r"(lstm_layer(?:_mc|_fused)?_kernel)I(Lb[01]E)", mangled)
    assert m, mangled
    fam = m.group(1)
    if fam == "lstm_layer_fused_kernel":
        fam += "<" + ("true" if m.group(2) == "Lb1E" else "false")
    return fam


@pytest.fixture(scope="module")
def built():
    from code_intelligence_b200 import _lib
    _lib.load()                                            # builds the library if needed
    return os.path.join(BUILD, "lstm_layer.ptxas.log"), os.path.join(BUILD, "lstm_layer.o")


@pytest.fixture(scope="module")
def sass(built):
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    text = subprocess.run([tool, "-sass", built[1]], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r"\n\s+Function : ", text)[1:]:
        name = chunk.split("\n", 1)[0].strip()
        if "lstm_layer" in name:
            funcs[name] = [re.sub(r"\s+", " ", l.split(";")[0]).strip() for l in chunk.split("\n")
                           if re.search(r"/\*[0-9a-f]{4,}\*/", l)]
    assert len(funcs) == 36, sorted(funcs)                 # 12 instantiations x 3 gate modes
    return funcs


def test_ptxas_applied_setmaxnreg_and_spills_stay_within_design_figures(built):
    text = open(built[0]).read()
    assert "C7507" not in text, "ptxas ignored setmaxnreg in some recurrent kernel"
    blocks = re.split(r"ptxas info\s+: Compiling entry function '", text)[1:]
    seen = 0
    for b in blocks:
        name = b.split("'", 1)[0]
        if "lstm_layer" not in name:
            continue
        seen += 1
        regs = int(re.search(r"Used (\d+) registers", b).group(1))
        spill = int(re.search(r"(\d+) bytes spill stores", b).group(1))
        # the launch must hand out exactly the 168 registers the setmaxnreg budgets (40 / 232) redistribute
        assert regs == 168, (name, regs)
        assert spill <= SPILL_LIMITS[_demangled_family(name)], (name, spill)
    assert seen == 36


def test_every_recurrent_kernel_moves_registers_to_the_consumers(sass):
    for name, lines in sass.items():
        alloc = [l for l in lines if "USETMAXREG.TRY_ALLOC" in l]
        dealloc = [l for l in lines if "USETMAXREG.DEALLOC" in l]
        assert alloc and all(l.endswith("0xe8") for l in alloc), (name, alloc)        # 232
        assert dealloc and all(l.endswith("0x28") for l in dealloc), (name, dealloc)  # 40


def test_consumer_k_loop_has_no_local_memory_and_loads_miss_the_accumulators(sass):
    """Consumer K loop (from the consumers' first full-barrier wait to the final wgmma wait, with the early loads of
    the epilogue inputs): no LDL / STL, and no global load writes a register of the wgmma accumulator block while
    MMAs may be in flight."""
    for name, lines in sass.items():
        alloc = next(i for i, l in enumerate(lines) if "USETMAXREG.TRY_ALLOC" in l)
        start = next(i for i in range(alloc, len(lines)) if "SYNCS.PHASECHK" in lines[i])
        end = next(i for i in range(start, len(lines)) if "WARPGROUP.DEPBAR.LE gsb0, 0x0" in lines[i])
        region = lines[start:end]
        assert not [l for l in region if re.search(r"\b(LDL|STL)\b", l)], name
        acc = {int(m.group(1)) for l in region for m in [re.search(r"HGMMA\S* R(\d+),", l)] if m}
        assert len(acc) == 1, (name, acc)
        lo = acc.pop()
        hi = lo + 128
        loads = [l for l in region if re.search(r"\bLDG\b|\bLDG\.", l)]
        assert loads, name
        for l in loads:
            dst = int(re.search(r"LDG\S* R(\d+)", l).group(1))
            assert not (lo - 3 <= dst < hi), (name, l, lo)   # a 128-bit load writes dst .. dst + 3
