"""The page kernel has one instance per output layout (model_kernels.cuh MODEL_LAYOUTS), read out of the built library
without a GPU (`cuobjdump -res-usage`): every layout a call can ask for must exist for both models, and each instance must
keep the occupancy DESIGN.md argues from -- 8 blocks of 256 threads per SM for BPE (7 for WordPiece's longer halo).
The headline's layout (BPE, ids + char offsets) must not use more local memory than the single runtime-flag instance
it replaced (32 B stack on sm_90a, all of it from the look-up and merge phases)."""
import os, re, shutil, subprocess
import pytest
from helpers import ROOT

LIB = os.path.join(ROOT, "tokenizers_b200", "libb2t.so")
# L_OFFSETS 1, L_WORD_IDS 2, L_BYTE_OFFSETS 4, L_PREFIX 8, L_ADDED_IDS 16; byte offsets and the prefix mapping only with offsets
LAYOUTS = sorted(m for m in range(32) if not (m & 12) or (m & 1))


def _res():
    if shutil.which("cuobjdump") is None or not os.path.exists(LIB):
        pytest.skip("cuobjdump or libb2t.so not available")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    res = {}
    for m in re.finditer(r"Function _ZN3b2t17model_tile_kernelILi(\d)ELj(\d+)E\S*:\n\s+REG:(\d+) STACK:(\d+) SHARED:(\d+)", out):
        res[(int(m.group(1)), int(m.group(2)))] = tuple(int(x) for x in m.groups()[2:])
    return res


def test_every_layout_has_an_instance():
    res = _res()
    assert len(LAYOUTS) == 20
    for model in (0, 1):
        assert sorted(l for (m, l) in res if m == model) == LAYOUTS, model


def test_every_instance_fits_its_blocks_per_sm():
    for (model, lay), (reg, stack, shared) in _res().items():
        blocks = 8 if model == 0 else 7
        assert reg <= 32, (model, lay, reg)
        # SHARED as cuobjdump reports it includes the 1 KB per block the system reserves; an SM has 228 KB
        assert shared * blocks <= 233472, (model, lay, shared)
        assert stack <= 32, (model, lay, stack)


def test_headline_layout():
    reg, stack, shared = _res()[(0, 1)]   # BPE, ids + char offsets
    assert reg <= 32 and shared * 8 <= 233472 and stack <= 32, (reg, stack, shared)
