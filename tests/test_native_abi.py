"""The C-ABI library loads and exports every symbol include/bnpk.h declares (no GPU, no compute)."""
import os
import re

from bionumpy_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "bnpk.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(bnpk_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = _native.load_library()
    names = declared_symbols()
    assert len(names) >= 20
    for name in names:
        assert hasattr(lib, name), f"{name} declared in include/bnpk.h but not exported"
    assert set(names) == set(_native.SIGNATURES), set(names) ^ set(_native.SIGNATURES)
    assert lib.bnpk_abi_version() == 3


def test_header_constants_match_python_mirror():
    text = open(os.path.join(ROOT, "include", "bnpk.h")).read()
    for name, val in (("BNPK_ENC_ASCII_ACGT", _native.ENC_ASCII_ACGT), ("BNPK_ENC_ASCII_ACTG", _native.ENC_ASCII_ACTG),
                      ("BNPK_ENC_CODES", _native.ENC_CODES), ("BNPK_ENC_LUT", _native.ENC_LUT),
                      ("BNPK_HIST_GLOBAL", _native.HIST_GLOBAL), ("BNPK_E_K", _native.E_K)):
        m = re.search(rf"#define\s+{name}\s+\(?(-?\d+)\)?", text)
        assert m and int(m.group(1)) == val, name
    for name, val in (("BNPK_ST_BAD_BASE", _native.ST_BAD_BASE), ("BNPK_ST_LAST_ROW_INDEX", _native.ST_LAST_ROW_INDEX),
                      ("BNPK_ST_WORDS", _native.ST_WORDS)):
        m = re.search(rf"{name}\s*=\s*(\d+)", text)
        assert m and int(m.group(1)) == val, name


def test_workspace_size_is_monotone():
    lib = _native.load_library()
    sizes = [lib.bnpk_tile_workspace_bytes(n) for n in (0, 1, 32768, 10 ** 6, 10 ** 9)]
    assert sizes == sorted(sizes) and sizes[0] >= 128


def test_compute_fails_loudly_without_gpu():
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("has a GPU")
    import bionumpy_b200 as bnp
    with pytest.raises(_native.NativeLibraryError):
        bnp.as_encoded_array("ACGT", bnp.DNAEncoding)
    with pytest.raises(_native.NativeLibraryError):
        bnp.get_kmers(bnp.as_encoded_array("ACGT"), 3)
    with pytest.raises(_native.NativeLibraryError):
        bnp.FastQBuffer.from_raw_buffer(bnp.as_encoded_array("@a\nACGT\n+\n!!!!\n"))


def test_torch_library_registers_the_ops():
    """libbnpk_torch.so (TORCH_LIBRARY(bnpk, ...)) loads without a GPU and registers the dispatcher ops."""
    import torch
    from bionumpy_b200 import torch_ops
    ops = torch_ops.load()
    for name in ("chunk_kmer_count", "line_split", "row_offsets", "rows_encode", "rows_kmer_hash", "rows_kmer_count",
                 "rows_reverse_complement", "bincount"):
        assert hasattr(ops, name), name
    schema = torch._C._get_schema("bnpk::chunk_kmer_count", "")
    assert "Tensor(a!) hist" in str(schema)


def test_dominant_kernels_are_sm90a_code_without_spills():
    """The in-tree library carries sm_90a SASS of both builds of the warp-specialised kernel, within the register budget
    of their CTA sizes (576 and 704 threads) and without local-memory spills (cuobjdump works without a GPU)."""
    import shutil
    import subprocess
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        import pytest
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", _native.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    blocks = out.split(" Function ")
    seen = {}
    for name, regs_max in (("_ZN4bnpk2ws14tile_ws_kernelILi0EEEvNS_8TileArgsE", 112), ("_ZN4bnpk3wsm14tile_ws_kernelILi0EEEvNS_8TileArgsE", 88)):
        blk = next(b for b in blocks if b.startswith(name))
        m = re.search(r"REG:(\d+) STACK:(\d+)", blk)
        assert m, blk[:200]
        seen[name] = (int(m.group(1)), int(m.group(2)))
        assert int(m.group(1)) <= regs_max and int(m.group(2)) == 0, (name, m.group(0))
    assert len(seen) == 2


def _python_sources(path):
    for dirpath, _, files in os.walk(path):
        for f in sorted(files):
            if f.endswith(".py"):
                yield os.path.join(dirpath, f)


def test_only_the_bindings_call_the_library():
    """Every call of libbnpk.so from the package goes through ops.py, which checks its tensors, or _native.py: no other
    module names a bnpk_* symbol.  In ops.py, only the one tensor rule (_pointer) makes pointers and only _on_device
    switches the device."""
    import ast
    pkg = os.path.join(ROOT, "bionumpy_b200")
    found = []
    for path in _python_sources(pkg):
        if os.path.basename(path) in ("ops.py", "_native.py") and os.path.dirname(path) == pkg:
            continue
        for node in ast.walk(ast.parse(open(path).read())):
            name = getattr(node, "attr", None) or getattr(node, "id", None) or ""
            if isinstance(node, ast.Constant) and isinstance(node.value, str):
                name = node.value
            if re.fullmatch(r"bnpk_\w+", name):
                found.append(f"{os.path.relpath(path, ROOT)}:{node.lineno} {name}")
    assert not found, found
    tree = ast.parse(open(os.path.join(pkg, "ops.py")).read())
    methods = [m for c in tree.body if isinstance(c, ast.ClassDef) for m in c.body]
    for fn in [f for f in tree.body + methods if isinstance(f, ast.FunctionDef)]:
        for node in ast.walk(fn):
            if isinstance(node, ast.Call):
                callee = ast.unparse(node.func)
                assert callee != "ptr" or fn.name == "_pointer", f"ptr() in {fn.name}"
                assert callee != "torch.cuda.device" or fn.name == "_on_device", f"a device switch in {fn.name}"
                assert not callee.endswith(".data_ptr"), f"data_ptr() in {fn.name}"
