"""The occupancy and instruction budgets DESIGN.md argues from, checked on the built library without a GPU
(`cuobjdump` reads them out of libb2t.so): the page kernel must fit 8 blocks of 256 threads per SM (32 registers,
<= 28.5 KB of shared memory each; the WordPiece variant with its longer halo 7), the lean scan kernels 8 blocks of 128
threads (64 registers), the Llama-3 scan kernel 4 (128 registers), and the lean scan's static instruction count must
not creep up -- it is bound by instruction issue (DESIGN.md §8).  The static counts are those of the sm_90a build."""
import os, re, shutil, subprocess
import pytest
from helpers import ROOT

LIB = os.path.join(ROOT, "tokenizers_b200", "libb2t.so")


def _res():
    if shutil.which("cuobjdump") is None or not os.path.exists(LIB):
        pytest.skip("cuobjdump or libb2t.so not available")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    res = {}
    for m in re.finditer(r"Function (\S+):\n\s+REG:(\d+) STACK:(\d+) SHARED:(\d+)", out):
        res[m.group(1)] = tuple(int(x) for x in m.groups()[1:])
    return res


def test_page_kernel_fits_eight_blocks_per_sm():
    res = _res()
    # SHARED as cuobjdump reports it includes the 1 KB per block the system reserves; an SM has 228 KB
    for model, blocks in ((0, 8), (1, 7)):  # BPE: 8 blocks per SM; WordPiece (416-byte halo): 7
        reg, stack, shared = next(v for k, v in res.items() if f"model_tile_kernelILi{model}E" in k)
        assert reg <= 32, "8 blocks x 256 threads need <= 32 registers per thread (64 K registers per SM)"
        assert shared * blocks <= 233472, f"{blocks} blocks per SM need <= {233472 // blocks} bytes of shared memory each"
        assert stack <= 64


def test_llama3_stream_kernel_registers_and_stack():
    """The Llama-3 scan (window algebra, two iterations of class masks live) runs 4 blocks of 128 threads per SM."""
    res = _res()
    for added in (0, 1):
        reg, stack, shared = next(v for k, v in res.items() if f"pretok_stream_kernelILi1ELb{added}E" in k)
        assert reg <= 128, "4 blocks x 128 threads need <= 128 registers per thread (64 K registers per SM)"
        assert shared <= 1024, "no shared memory"
        assert stack <= 64, "a few words of local memory for the rare slow path (sm_90a: 40 B)"


def test_streaming_scan_and_prepass_kernels():
    """Round 2: the streaming scan (the kernel the roofline figure is about) must stay at 8 blocks of 128 threads per SM without
    local memory and must not grow -- it is bound by the issue of its integer instructions (DESIGN.md §8);
    the added-token variants and the Bert variant share the budget; the normalizer pre-pass keeps 6 blocks of 256 threads."""
    res = _res()
    lean = {k: v for k, v in res.items() if "pretok_lean_kernel" in k}
    assert len(lean) >= 8, sorted(lean)          # GPT-2, Whitespace, no-regex, Bert, each with and without added-token bitmaps
    for k, (reg, stack, shared) in lean.items():
        assert reg <= 64 and stack == 0 and shared <= 1024, (k, reg, stack, shared)
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    body = sass.split("Function : _ZN3b2t18pretok_lean_kernelILi0ELb0E", 1)[1].split("Function : ", 1)[0]
    n = len(re.findall(r"^\s+/\*[0-9a-f]{4}\*/\s", body, flags=re.M))
    assert 500 < n <= 1000, f"{n} static instructions in the GPT-2 streaming scan (sm_90a: 944)"
    assert len(re.findall(r"\bLOP3\b", body)) <= 316, "boolean operations of the scan (sm_90a: 300 static)"
    reg, stack, shared = next(v for k, v in res.items() if "norm_write_kernel" in k)
    assert reg <= 40 and shared * 6 <= 233472, "6 blocks x 256 threads per SM"
    reg, stack, shared = next(v for k, v in res.items() if "norm_count_kernel" in k)
    assert reg <= 32
    for name in ("added_scan_kernel", "added_resolve_kernel", "dense_rows_kernel", "norm_offsets_kernel"):
        assert any(name in k for k in res), name
