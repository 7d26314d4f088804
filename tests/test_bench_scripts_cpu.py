"""The C4 query-form benchmark scripts (scripts/bench_c4*.py) and their shared harness (scripts/c4bench.py): the
scripts import the harness and never one another, the harness still generates the published workloads' clouds byte
for byte, and every script's command line keeps its defaults."""
import ast
import glob
import hashlib
import importlib.util
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = os.path.join(ROOT, "scripts")


def _c4bench():
    spec = importlib.util.spec_from_file_location("c4bench", os.path.join(SCRIPTS, "c4bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _bench_scripts():
    return sorted(glob.glob(os.path.join(SCRIPTS, "bench_c4*.py")))


def test_bench_scripts_do_not_import_each_other():
    for path in _bench_scripts():
        modules = []
        for node in ast.walk(ast.parse(open(path).read(), path)):
            if isinstance(node, ast.Import):
                modules += [a.name for a in node.names]
            elif isinstance(node, ast.ImportFrom):
                modules.append(node.module or "")
        assert not [m for m in modules if m.split(".")[0].startswith("bench_c4")], (os.path.basename(path), modules)


# SHA-256 of the fp32 CPU tensor bytes, from the functions these clouds were first published with
SCENE_DIGESTS = {
    (100_000, 200): "7e3363282bffa6264efdbdc8dcde9655ce2061ba28791ebf169cc4c0922009c8",
    (100_000, 201): "e6de7750c3120c3f9dd11bc1d6545821e03bd64402f28fb6183b016b601fabc6",
    (1_000_000, 300): "6f7c820f005dfaf32a6f4304546304a25329c5517c958b1f19b41f29ebca2fad",
    (1000, 7): "3ee4807b8f15be75d7fc1fb1f04399cd5ed275974efca4ae75cca9047ded7a8a",
}
CLOUD_DIGESTS = {
    ("uniform", 200, (10_000,), 300): "54ed29785813c04359f60549e48b4e0d1c29f45135f7415c35c04ddc0c57b16b",
    ("scene", 200, (10_000,), 300): "3f31ca66952320dbe8472d223e493485d69a5bcc1686f2f916df80f4d6c130e8",
    ("uniform", 1024, (8, 256), 301): "7f930d5d625d2e689c36fbae6bdb279b941a36d4201a7e1c026d110d8205eeff",
    ("scene", 1024, (8, 256), 301): "19bf1e3114b60e17bc0f37d59f51f1fea45014dd16f20a0a8cccb34a9848f57e",
    ("scene", 65_536, (64,), 300): "fa67ec32f42fb55511787e2d2ce607cb62f3ab41cec20ec247f23976582502a1",
}


def _digest(t, shape):
    import torch
    assert t.device.type == "cpu" and t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == shape
    return hashlib.sha256(t.numpy().tobytes()).hexdigest()


def test_workload_clouds_unchanged():
    c4 = _c4bench()
    for (n, seed), want in SCENE_DIGESTS.items():
        assert _digest(c4.scene_points(n, seed), (n, 3)) == want, (n, seed)
    for (kind, A, seg_shape, seed), want in CLOUD_DIGESTS.items():
        got = _digest(c4.clouds(kind, A, seg_shape, seed), (A, *seg_shape, 3))
        assert got == want, (kind, A, seg_shape, seed)


# every script's options and defaults, as README.md and DESIGN.md quote them
CLI_DEFAULTS = {
    "bench_c4tri.py": {"steps": "50", "warmup": "5", "rounds": "3", "n-cfg": "200", "n-pts": "100000"},
    "bench_c4prim.py": {"steps": "50", "warmup": "5", "rounds": "3", "n-cfg": "200", "n-pts": "100000"},
    "bench_c4paired.py": {"steps": "10", "warmup": "2", "rounds": "3", "shapes": "200x10000,4096x2048,65536x64"},
    "bench_c4swept.py": {"steps": "20", "warmup": "3", "rounds": "3"},
    "bench_c4clearance.py": {"steps": "20", "warmup": "3", "rounds": "3"},
    "bench_c4paired_clearance.py": {"steps": "20", "warmup": "3", "rounds": "3"},
    "bench_c4self_clearance.py": {"steps": "20", "warmup": "3", "rounds": "3"},
    "bench_c4collision_cost.py": {"steps": "10", "warmup": "2", "rounds": "2"},
    "bench_c4paired_collision_cost.py": {"steps": "10", "warmup": "2", "rounds": "3"},
    "bench_c4self_collision_cost.py": {"steps": "20", "warmup": "3", "rounds": "3"},
}


def test_bench_scripts_help_shows_defaults():
    assert sorted(CLI_DEFAULTS) == [os.path.basename(p) for p in _bench_scripts()]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", COLUMNS="200")
    procs = {name: subprocess.Popen([sys.executable, os.path.join(SCRIPTS, name), "--help"], cwd=ROOT, env=env,
                                    stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for name in CLI_DEFAULTS}
    for name, proc in procs.items():
        out, _ = proc.communicate(timeout=300)
        assert proc.returncode == 0, (name, out)
        options = dict(re.findall(r"^\s*--([\w-]+) \S+\s.*\(default: ([^)]*)\)$", out, re.M))
        assert options == CLI_DEFAULTS[name], (name, out)
