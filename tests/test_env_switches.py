"""Every environment variable the package reads, in one list.  Each kernel dispatch has one code path (the one the benchmarks and the GPU
tests run); a variable that selects another path would keep code alive that nothing exercises.  Adding a variable means adding it here and to
the README's list."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "nabladft_b200")

ALLOWED = {
    "NB200_GOC_GEMM",        # =simt: GemNet-OC dense layers on the functor GEMM (tells kernel faults from GEMM-dispatch faults)
    "NB200_TRAIN_STORAGE",   # default per-edge storage of the training arrays (a precision choice, INTEGRATION.md)
    "NB200_QH_PAIR_CHUNK",   # QHNet memory bound: atom pairs whose path weights exist at a time
    "NVCC",                  # build: compiler
    "NB200_NVCC_EXTRA",      # build: extra flags
}

C_READ = re.compile(r"\bgetenv\s*\(")
C_KEY = re.compile(r"\bgetenv\s*\(\s*\"([^\"]+)\"\s*\)")
PY_READ = re.compile(r"\bos\.(?:environ\b|getenv\s*\()")
PY_KEY = re.compile(r"\bos\.(?:environ\.get\s*\(|environ\s*\[|getenv\s*\()\s*[\"']([^\"']+)[\"']")


def _reads(files, read, key):
    keys, unresolved = set(), []
    for path in files:
        with open(path) as f:
            for n, line in enumerate(f, 1):
                found = key.findall(line)
                keys.update(found)
                if len(read.findall(line)) != len(found):
                    unresolved.append(f"{os.path.relpath(path, ROOT)}:{n}: {line.strip()}")
    return keys, unresolved


def test_environment_variables_are_exactly_the_allowlist():
    csrc = [p for ext in ("cu", "cuh", "inc", "h") for p in glob.glob(os.path.join(PKG, "csrc", f"*.{ext}"))]
    assert csrc, "no CUDA sources found"
    c_keys, c_bad = _reads(csrc, C_READ, C_KEY)
    py_keys, py_bad = _reads(glob.glob(os.path.join(PKG, "*.py")), PY_READ, PY_KEY)
    assert not c_bad + py_bad, "environment reads whose name is not a string literal:\n" + "\n".join(c_bad + py_bad)
    assert c_keys | py_keys == ALLOWED
