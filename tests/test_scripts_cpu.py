"""The measurement scripts under scripts/ without a GPU: every one imports and answers --help, the card query in
scripts/measure.py never raises, and every profile script measures through scripts/measure.py rather than its own copy
of a timer, a graph capture, an alternation loop or an nvidia-smi query."""
import ast
import glob
import importlib
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = sorted(glob.glob(os.path.join(ROOT, "scripts", "*.py")))
NAMES = [os.path.basename(p)[:-3] for p in SCRIPTS]
# two run under torchrun, and hrnn_train_check runs on the GPU as it is imported
CHECKERS = {"meta_dist_check", "hrnn_dist_check", "hrnn_train_check"}
IMPORTABLE = [n for n in NAMES if n not in CHECKERS]
PROFILES = [n for n in IMPORTABLE if n != "measure"]
WITH_CLI = [n for n in NAMES if "argparse" in open(os.path.join(ROOT, "scripts", n + ".py")).read()]

# what measure.py does once; a script defining any of these names has its own copy
OWN_HELPERS = {"card", "gpu_info", "timed", "time_ms", "time_calls", "event_ms", "graphed", "graph_ms", "wall_ms",
               "alternate", "summary", "emit"}
# clocks and graph capture are measure.py's; segmented_bptt_profile times the recomputes nested inside one backward,
# which no helper does
TIMING = {"Event", "CUDAGraph", "graph", "perf_counter", "time"}
NESTED_EVENTS = {("segmented_bptt_profile", "timed_recompute", "Event")}


def tree(name):
    with open(os.path.join(ROOT, "scripts", name + ".py")) as f:
        return ast.parse(f.read())


def functions(t):
    """(function name, node) for every node, the name of the innermost enclosing function ("" at module level)."""
    out = []

    def walk(node, fn):
        for child in ast.iter_child_nodes(node):
            inner = child.name if isinstance(child, (ast.FunctionDef, ast.AsyncFunctionDef)) else fn
            out.append((inner, child))
            walk(child, inner)
    walk(t, "")
    return out


def test_script_list():
    assert "measure" in NAMES and "tc_ab" in NAMES
    assert CHECKERS <= set(NAMES)
    assert set(WITH_CLI) >= set(PROFILES) - {"tc_accuracy", "tc_accuracy_large"}


@pytest.mark.parametrize("name", IMPORTABLE)
def test_imports_without_gpu(name):
    importlib.import_module("scripts." + name)


@pytest.mark.parametrize("name", WITH_CLI)
def test_help(name, tmp_path):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", name + ".py"), "--help"], cwd=tmp_path,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert "usage:" in r.stdout


@pytest.fixture
def fake_device(monkeypatch):
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(torch.cuda, "get_device_name", lambda device=None: "Fake GPU")


def fake_smi(tmp_path, body):
    p = tmp_path / "nvidia-smi"
    p.write_text("#!/bin/sh\n" + body + "\n")
    p.chmod(0o755)
    return str(tmp_path)


def test_card_reads_the_current_device(fake_device, tmp_path, monkeypatch):
    from scripts import measure
    log = tmp_path / "argv"
    monkeypatch.setenv("PATH", fake_smi(tmp_path, 'echo "$@" > %s\necho "NVIDIA H100 80GB HBM3, 700.00 W, 1980 MHz"'
                                        % log))
    assert measure.card() == {"device": "Fake GPU", "nvidia_smi": "NVIDIA H100 80GB HBM3, 700.00 W, 1980 MHz"}
    assert log.read_text().split() == ["--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                                       "-i", "0"]


def test_card_without_nvidia_smi(fake_device, monkeypatch):
    from scripts import measure
    monkeypatch.setenv("PATH", "")
    c = measure.card()
    assert set(c) == {"device", "nvidia_smi"} and c["device"] == "Fake GPU"
    assert c["nvidia_smi"].startswith("nvidia-smi failed")


def test_card_when_nvidia_smi_fails(fake_device, tmp_path, monkeypatch):
    from scripts import measure
    monkeypatch.setenv("PATH", fake_smi(tmp_path, "echo 'No devices were found' >&2\nexit 6"))
    c = measure.card()
    assert set(c) == {"device", "nvidia_smi"} and c["device"] == "Fake GPU"
    assert c["nvidia_smi"].startswith("nvidia-smi failed") and "No devices were found" in c["nvidia_smi"]


def test_only_measure_runs_nvidia_smi():
    for name in NAMES:
        if name == "measure":
            continue
        consts = [n.value for n in ast.walk(tree(name)) if isinstance(n, ast.Constant) and isinstance(n.value, str)]
        assert not [c for c in consts if c == "nvidia-smi" or c.startswith("nvidia-smi ")], name


@pytest.mark.parametrize("name", PROFILES)
def test_profiles_measure_through_measure_py(name):
    for fn, node in functions(tree(name)):
        if isinstance(node, (ast.FunctionDef, ast.AsyncFunctionDef)):
            assert node.name not in OWN_HELPERS, (name, node.name)
        if isinstance(node, ast.Attribute) and node.attr in TIMING:
            assert (name, fn, node.attr) in NESTED_EVENTS, (name, fn, node.attr, node.lineno)


@pytest.mark.parametrize("name", PROFILES)
def test_profiles_import_no_other_profile(name):
    others = set(NAMES) - {"measure", name}
    for node in ast.walk(tree(name)):
        if isinstance(node, ast.ImportFrom) and node.module:
            mods = [node.module] + [node.module + "." + a.name for a in node.names]
        elif isinstance(node, ast.Import):
            mods = [a.name for a in node.names]
        else:
            continue
        for m in mods:
            parts = m.split(".")
            assert not (parts[0] in others or (parts[0] == "scripts" and len(parts) > 1 and parts[1] in others)), \
                (name, m)
