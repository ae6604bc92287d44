"""Every GRB_* environment switch the native code reads is exercised by a GPU test, or is listed here with the reason
it is not.  A switch added later without a test fails this (CPU) test."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE_DIRS = (os.path.join("granite_b200", "csrc"), os.path.join("granite_b200", "host"))
SOURCE_EXTS = (".cu", ".cuh", ".cpp", ".hpp", ".h", ".inc")
GETENV = re.compile(r'getenv\(\s*"(GRB_[A-Z0-9_]+)"\s*\)')

ALLOWED_UNTESTED = {
    "GRB_HOST_PROFILE": "prints host-side timings only; no computed value depends on it",
}


def switches_read(root):
    """{switch: [source files reading it]} for every getenv("GRB_...") under root's native source directories."""
    found = {}
    for sub in SOURCE_DIRS:
        for dirpath, _, files in os.walk(os.path.join(root, sub)):
            for name in sorted(files):
                if not name.endswith(SOURCE_EXTS):
                    continue
                path = os.path.join(dirpath, name)
                with open(path, encoding="utf-8", errors="replace") as fh:
                    for sw in GETENV.findall(fh.read()):
                        found.setdefault(sw, []).append(os.path.relpath(path, root))
    return found


def gpu_test_sources(tests_dir):
    """Text of the GPU test modules (marked gpu) and of the worker modules they start in child processes."""
    texts = []
    for name in sorted(os.listdir(tests_dir)):
        if not name.endswith(".py") or name == os.path.basename(__file__):
            continue
        with open(os.path.join(tests_dir, name), encoding="utf-8") as fh:
            text = fh.read()
        if name.endswith("_worker.py") or (name.startswith("test_") and "pytest.mark.gpu" in text):
            texts.append(text)
    return texts


def untested_switches(root, tests_dir, allowed):
    """Switches read under root that no GPU test names and `allowed` does not list."""
    texts = gpu_test_sources(tests_dir)
    return sorted(sw for sw in switches_read(root) if sw not in allowed and not any(sw in t for t in texts))


def test_every_switch_has_a_gpu_test():
    read = switches_read(ROOT)
    assert "GRB_POST_EXACT" in read and "GRB_NO_ASYNC_POST" in read, "the scan must find the known switches"
    missing = untested_switches(ROOT, os.path.join(ROOT, "tests"), ALLOWED_UNTESTED)
    assert not missing, f"switches read by the native code but named in no GPU test: {missing} ({ {k: read[k] for k in missing} })"


def test_allow_list_names_only_switches_that_exist():
    stale = sorted(set(ALLOWED_UNTESTED) - set(switches_read(ROOT)))
    assert not stale, f"allow-listed switches no longer read anywhere: {stale}"


def test_an_unlisted_switch_is_reported(tmp_path):
    src = tmp_path / "granite_b200" / "csrc"
    src.mkdir(parents=True)
    (src / "k.cu").write_text('static const bool a = getenv("GRB_X") != nullptr;\nstatic const bool b = getenv("GRB_HOST_PROFILE") != nullptr;\n')
    host = tmp_path / "granite_b200" / "host"
    host.mkdir()
    (host / "h.cpp").write_text('const char *e = std::getenv("GRB_Y");\n')
    tests = tmp_path / "tests"
    tests.mkdir()
    (tests / "test_y_gpu.py").write_text('import pytest\npytestmark = pytest.mark.gpu\nENV = {"GRB_Y": "1"}\n')
    (tests / "test_x_cpu.py").write_text('ENV = {"GRB_X": "1"}  # a CPU test does not count\n')
    assert switches_read(str(tmp_path)) == {"GRB_X": ["granite_b200/csrc/k.cu"], "GRB_HOST_PROFILE": ["granite_b200/csrc/k.cu"], "GRB_Y": ["granite_b200/host/h.cpp"]}
    assert untested_switches(str(tmp_path), str(tests), ALLOWED_UNTESTED) == ["GRB_X"]
