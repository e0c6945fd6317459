"""ORACLE (test infrastructure, NOT product code): the SASS of a built object, read with cuobjdump, for tests that pin
the instruction order an exact restatement relies on (tests/test_language_model_reference.py,
tests/test_lm_generation_reference.py)."""
from __future__ import annotations

import os
import re
import shutil
import subprocess


def sass_functions(obj):
    """{function name: [(opcode, operands, line)]} of cuobjdump -sass, predicates dropped.  Skips the calling test
    when cuobjdump is not installed."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        import pytest
        pytest.skip("cuobjdump is not installed")
    text = subprocess.run([exe, "-sass", obj], capture_output=True, text=True, check=True).stdout
    out = {}
    for block in re.split(r"\n\s*Function : ", text)[1:]:
        name = block.split("\n", 1)[0].strip()
        out[name] = [(m.group(1), m.group(2).strip(), m.group(0)) for m in
                     re.finditer(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)\s*([^;]*);[^\n]*", block)]
    return out
