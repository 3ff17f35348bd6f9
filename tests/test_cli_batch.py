"""The CLI's hidden --input_list: many images in one process, each group's Y planes through one collection-chain call.
Every output must be byte for byte the PNG the single-image CLI writes for that input with the same flags; the checks before any
work (-o, the list, clashing outputs) must exit with 1 and write nothing."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT

cv2 = pytest.importorskip("cv2")
PKG = os.path.join(ROOT, "waifu2x-converter-cpp_b200")
CLI = os.path.join(PKG, "w2x-converter")
MULTI_ENV = {"CUDA_DEVICE_MAX_CONNECTIONS": "32", "CUDA_MODULE_LOADING": "EAGER"}   # two contexts of one device side by side
# (w, h): 1-pixel sides, odd sizes, and 700x500, which the single-image path converts in blocks
SIZES = [(1, 1), (2, 3), (1, 40), (40, 1), (45, 33), (17, 29), (31, 8), (64, 47), (9, 100), (33, 65), (128, 3), (700, 500)]
MODES = {
    "noise1": ["-m", "noise", "--noise_level", "1"],
    "noise2": ["-m", "noise", "--noise_level", "2"],
    "scale2": ["-m", "scale", "--scale_ratio", "2.0"],
    "scale3": ["-m", "scale", "--scale_ratio", "3.0"],
    "scale1.6": ["-m", "scale", "--scale_ratio", "1.6"],
    "scale4": ["-m", "scale", "--scale_ratio", "4.0"],
    "scale1": ["-m", "scale", "--scale_ratio", "1.0"],
    "noise_scale": ["-m", "noise_scale"],
    "tta": ["-m", "noise_scale", "--tta", "1"],
}


@pytest.fixture(scope="module")
def cli(w2x):
    w2x.build()
    assert os.path.exists(CLI)
    return CLI


def _image(w, h, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    img = np.stack([128 + 100 * np.sin(xx / 5.0 + c + seed) * np.cos(yy / 4.0 - c) for c in range(3)], -1) + rng.normal(0, 12, (h, w, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


def _run(*args, cwd=None, env=None):
    return subprocess.run([CLI, *args], capture_output=True, text=True, cwd=cwd, env=dict(os.environ, **(env or {})))


def _auto_suffix(args):
    """the part the (auto) rule appends to an input name without its extension"""
    opt = dict(zip(args[::2], args[1::2]))
    mode, level, ratio = opt.get("-m", "noise_scale"), opt.get("--noise_level", "1"), float(opt.get("--scale_ratio", "2.0"))
    s = f"({mode})"
    if "noise" in mode:
        s += f"(Level{level})"
    if "scale" in mode:
        s += f"(x{ratio:.6f})"
    return s + ".png"


class Inputs:
    """the images, in two directories (and one in the working directory itself), with the single-image CLI's PNG per mode"""

    def __init__(self, root, model_dir):
        self.root, self.model_dir = root, model_dir
        self.names = []
        for i, (w, h) in enumerate(SIZES):
            rel = os.path.join("a" if i % 3 == 0 else "b" if i % 3 == 1 else "", f"img{i}.png")
            os.makedirs(os.path.join(root, os.path.dirname(rel)), exist_ok=True)
            cv2.imwrite(os.path.join(root, rel), _image(w, h, i))
            self.names.append(rel)
        self._refs = {}

    def write_list(self, path, names=None, sep="\n"):
        with open(path, "w", newline="") as f:
            f.write(sep.join(names if names is not None else self.names) + sep)
        return path

    def refs(self, mode):
        """{input: bytes of the single-image CLI's output} for one mode, every image converted by its own process"""
        if mode not in self._refs:
            d = os.path.join(self.root, "ref_" + mode)
            os.makedirs(d)
            out = {}
            for i, name in enumerate(self.names):
                r = _run("-i", name, "-o", os.path.join(d, f"{i}.png"), "--model_dir", self.model_dir, *MODES[mode], cwd=self.root)
                assert r.returncode == 0, (mode, name, r.stdout + r.stderr)
                with open(os.path.join(d, f"{i}.png"), "rb") as f:
                    out[name] = f.read()
            self._refs[mode] = out
        return self._refs[mode]

    def batch(self, mode, out_dir, extra=(), env=None, names=None):
        """one --input_list run into out_dir; returns the run and {input: bytes of its output}"""
        os.makedirs(out_dir)
        lst = self.write_list(os.path.join(out_dir, "..", os.path.basename(out_dir) + ".txt"), names)
        r = _run("--input_list", lst, "-o", out_dir, "--model_dir", self.model_dir, *MODES[mode], *extra, cwd=self.root, env=env)
        got = {}
        for name in names if names is not None else self.names:
            p = os.path.join(out_dir, os.path.splitext(os.path.basename(name))[0] + _auto_suffix(MODES[mode]))
            if os.path.exists(p):
                with open(p, "rb") as f:
                    got[name] = f.read()
        return r, got


@pytest.fixture(scope="module")
def inputs(cli, json_models, tmp_path_factory):
    return Inputs(str(tmp_path_factory.mktemp("batch")), os.path.dirname(json_models["scale2.0x"]))


def _check_identical(inputs, mode, got):
    ref = inputs.refs(mode)
    assert sorted(got) == sorted(ref), mode
    for name in ref:
        assert got[name] == ref[name], (mode, name)


def _stdout_lines(names, out_of):
    return [f"{n} -> {out_of(n)}" for n in names] + ["process successfully done!"]


# ---- the GPU ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_batch_writes_the_single_image_png(inputs, mode):
    r, got = inputs.batch(mode, os.path.join(inputs.root, "out_" + mode), extra=["-j", "3"])
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.splitlines()[-1] == "process successfully done!"
    assert "Iteration #" not in r.stdout and "scaling" not in r.stdout        # no per-layer or per-pass progress lines
    _check_identical(inputs, mode, got)


def _groups(sizes, upscales, tta, budget):
    """the grouping rule restated: a group closes before the image that would take its cost past the budget"""
    groups, cost = 0, 0
    for w, h in sizes:
        c = (w * h << (2 * upscales)) * (8 if tta else 1)
        if groups == 0 or cost + c > budget:
            groups, cost = groups + 1, c
        else:
            cost += c
    return groups


@pytest.mark.gpu
@pytest.mark.parametrize("mode,budget", [("noise_scale", 30000), ("tta", 150000), ("noise1", 3000)])
def test_groups_change_nothing_but_the_grouping(inputs, mode, budget):
    upscales = 1 if "scale" in MODES[mode][1] else 0
    tta = "--tta" in MODES[mode]
    expect = _groups(SIZES, upscales, tta, budget)
    assert expect >= 3 and (SIZES[-1][0] * SIZES[-1][1] << 2 * upscales) * (8 if tta else 1) > budget   # 700x500 forms a group alone
    r, got = inputs.batch(mode, os.path.join(inputs.root, f"groups_{mode}"), env={"W2X_CLI_BATCH_PIXELS": str(budget), "W2X_CLI_TIMING": "1"})
    assert r.returncode == 0, r.stdout + r.stderr
    m = re.search(r'\{"w2x_cli_batch_timing_ms": \{"images": (\d+), "groups": (\d+), "convert": [0-9.e+-]+, "total": [0-9.e+-]+\}\}', r.stderr)
    assert m, r.stderr
    assert (int(m.group(1)), int(m.group(2))) == (len(SIZES), expect)
    _check_identical(inputs, mode, got)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["noise_scale", "tta", "scale4"])
def test_two_gpus_write_the_one_gpu_single_image_png(inputs, mode):
    """W2X_DEVICES=0,0: whole images and TTA variants spread over two contexts; --tta 1 works here, unlike for one image"""
    r, got = inputs.batch(mode, os.path.join(inputs.root, f"multi_{mode}"), env=dict(MULTI_ENV, W2X_DEVICES="0,0"))
    assert r.returncode == 0, r.stdout + r.stderr
    _check_identical(inputs, mode, got)


@pytest.mark.gpu
def test_stdout_and_auto_names_with_and_without_an_output_directory(inputs, tmp_path):
    mode = "scale2"
    ref = inputs.refs(mode)
    work = tmp_path / "work"
    for name in inputs.names:
        os.makedirs(os.path.dirname(work / name), exist_ok=True)
        shutil.copy(os.path.join(inputs.root, name), work / name)
    out_of = lambda n: os.path.splitext(n)[0] + _auto_suffix(MODES[mode])   # noqa: E731  (next to its input)
    inputs.write_list(str(work / "list.txt"), sep="\r\n")                   # CRLF list
    r = _run("--input_list", "list.txt", "--model_dir", inputs.model_dir, *MODES[mode], cwd=work)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.splitlines() == _stdout_lines(inputs.names, out_of)
    for name in inputs.names:
        assert (work / out_of(name)).read_bytes() == ref[name], name
    # -o <dir>: the last path component of each (auto) name, in that directory (given with a trailing slash)
    (work / "o").mkdir()
    r = _run("--input_list", "list.txt", "-o", "o/", "--model_dir", inputs.model_dir, *MODES[mode], cwd=work)
    assert r.returncode == 0, r.stdout + r.stderr
    out_o = lambda n: "o/" + os.path.basename(out_of(n))                     # noqa: E731
    assert r.stdout.splitlines() == _stdout_lines(inputs.names, out_o)
    assert sorted(os.listdir(work / "o")) == sorted(os.path.basename(out_of(n)) for n in inputs.names)
    for name in inputs.names:
        assert (work / out_o(name)).read_bytes() == ref[name], name


@pytest.mark.gpu
def test_an_unreadable_entry_is_skipped_and_the_run_fails(inputs, tmp_path):
    mode = "noise_scale"
    ref = inputs.refs(mode)
    with open(os.path.join(inputs.root, "garbage.png"), "wb") as f:
        f.write(b"not an image")
    names = inputs.names[:4] + ["missing.png"] + inputs.names[4:7] + ["garbage.png"] + inputs.names[7:]
    r, got = inputs.batch(mode, os.path.join(inputs.root, "bad_entry"), names=names)
    assert r.returncode == 255, r.stdout + r.stderr
    assert "process successfully done!" not in r.stdout
    assert "Error : couldn't read image missing.png (" in r.stderr and "Error : couldn't read image garbage.png (" in r.stderr
    assert sorted(got) == sorted(inputs.names)
    for name in inputs.names:
        assert got[name] == ref[name], name
    out_dir = os.path.join(inputs.root, "bad_entry")
    assert r.stdout.splitlines() == [f"{n} -> {out_dir}/{os.path.splitext(os.path.basename(n))[0]}{_auto_suffix(MODES[mode])}"
                                     for n in inputs.names]


# ---- no GPU needed -----------------------------------------------------------------------------------------------------------------
def test_input_list_is_hidden_and_exclusive_with_i(cli, tmp_path):
    h = _run("--help", cwd=tmp_path)
    assert h.returncode == 0 and "input_list" not in h.stdout and "--input_file" in h.stdout
    r = _run("-m", "noise", cwd=tmp_path)
    assert r.returncode == 1 and "input_file" in r.stderr and "input_list" not in r.stderr    # -i stays required, the usage unchanged
    (tmp_path / "list.txt").write_text("a.png\n")
    for args in (["-i", "a.png", "--input_list", "list.txt"], ["--input_list", "list.txt", "-i", "a.png"]):
        r = _run(*args, cwd=tmp_path)
        assert r.returncode == 1 and "PARSE ERROR" in r.stderr and "Mutually exclusive" in r.stderr, args
    assert _run("--input_list", "list.txt", "--input_list", "list.txt", cwd=tmp_path).returncode == 1
    assert sorted(os.listdir(tmp_path)) == ["list.txt"]


def test_checks_before_any_work_exit_1_and_write_nothing(cli, tmp_path):
    def run(*a):
        before = sorted(os.listdir(tmp_path))
        r = _run(*a, "--model_dir", "no_such_dir", cwd=tmp_path)   # a model would fail with 255: these stop before any is loaded
        assert r.returncode == 1 and r.stdout == "", (a, r.stdout + r.stderr)
        assert sorted(os.listdir(tmp_path)) == before, a
        return r.stderr
    cv2.imwrite(str(tmp_path / "x.png"), _image(5, 4, 1))
    os.makedirs(tmp_path / "d1")
    os.makedirs(tmp_path / "d2")
    cv2.imwrite(str(tmp_path / "d1" / "x.png"), _image(5, 4, 2))
    cv2.imwrite(str(tmp_path / "d2" / "x.png"), _image(5, 4, 3))
    assert "Error : couldn't open nope.txt" in run("--input_list", "nope.txt")
    (tmp_path / "empty.txt").write_text("\n\r\n\n")
    assert "empty.txt" in run("--input_list", "empty.txt")
    (tmp_path / "l.txt").write_text("x.png\n")
    assert "not a directory" in run("--input_list", "l.txt", "-o", "x.png")
    assert "not a directory" in run("--input_list", "l.txt", "-o", "no_such_dir")
    (tmp_path / "twice.txt").write_text("d1/x.png\nd2/x.png\n")
    err = run("--input_list", "twice.txt", "-o", "d1")
    assert "d1/x.png" in err and "d2/x.png" in err
    (tmp_path / "same.txt").write_text("x.png\n./x.png\n")                    # one file spelt two ways
    err = run("--input_list", "same.txt")
    assert "x.png and ./x.png" in err
    (tmp_path / "ext.txt").write_text("x.png\nx.ppm\n")                        # different inputs, one (auto) name
    assert "x.ppm" in run("--input_list", "ext.txt")
    bad_budget = subprocess.run([CLI, "--input_list", "l.txt"], capture_output=True, text=True, cwd=tmp_path,
                                env=dict(os.environ, W2X_CLI_BATCH_PIXELS="0"))
    assert bad_budget.returncode == 1 and "W2X_CLI_BATCH_PIXELS" in bad_budget.stderr


def test_a_missing_model_exits_255_before_any_image_is_read(cli, tmp_path):
    (tmp_path / "l.txt").write_text("missing.png\n")
    r = _run("--input_list", "l.txt", "--model_dir", "no_such_dir", cwd=tmp_path)
    assert r.returncode == 255 and "couldn't open no_such_dir/noise1_model.json" in r.stderr
    assert "couldn't read image" not in r.stderr and r.stdout == ""


@pytest.mark.parametrize("mode", ["noise", "scale", "noise_scale"])
def test_without_a_device_nothing_is_written(cli, tmp_path, json_models, mode):
    for i in range(3):
        cv2.imwrite(str(tmp_path / f"in{i}.png"), _image(24 + i, 20, i))
    (tmp_path / "l.txt").write_bytes(b"in0.png\r\n\r\nmissing.png\r\nin1.png\r\nin2.png")   # CRLF, a blank line, no final newline
    r = subprocess.run([CLI, "--input_list", "l.txt", "-m", mode, "--model_dir", os.path.dirname(json_models["scale2.0x"])],
                       capture_output=True, text=True, cwd=tmp_path, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode != 0 and "process successfully done!" not in r.stdout and r.stdout == ""
    assert sorted(os.listdir(tmp_path)) == ["in0.png", "in1.png", "in2.png", "l.txt"]
    assert "Error : couldn't read image missing.png (" in r.stderr                  # the path without its \r


@pytest.mark.parametrize("ratio", ["1.0", "0.75", "0.5"])
def test_images_without_a_gpu_step_get_the_single_image_host_passes(cli, tmp_path, json_models, ratio):
    """-m scale at a ratio <= 1 runs no GPU step, in one image's run or many (here without a device)"""
    mdir = os.path.dirname(json_models["scale2.0x"])
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    names = []
    for i, (w, h) in enumerate([(1, 1), (7, 3), (45, 33), (300, 200)]):
        names.append(f"in{i}.png")
        cv2.imwrite(str(tmp_path / names[-1]), _image(w, h, i))
    (tmp_path / "ref").mkdir()
    for n in names:
        r = subprocess.run([CLI, "-i", n, "-o", f"ref/{n}", "-m", "scale", "--scale_ratio", ratio, "--model_dir", mdir],
                           capture_output=True, text=True, cwd=tmp_path, env=env)
        assert r.returncode == 0, r.stdout + r.stderr
    (tmp_path / "l.txt").write_text("\n".join(names) + "\n")
    suffix = f"(scale)(x{float(ratio):.6f}).png"
    for budget in (None, 50):                                             # one group; groups of [1, 7x3], [45x33], [300x200]
        out = tmp_path / f"out{budget}"
        out.mkdir()
        benv = dict(env, W2X_CLI_TIMING="1", **({"W2X_CLI_BATCH_PIXELS": str(budget)} if budget else {}))
        r = subprocess.run([CLI, "--input_list", "l.txt", "-o", out.name, "-m", "scale", "--scale_ratio", ratio, "--model_dir", mdir, "-j", "2"],
                           capture_output=True, text=True, cwd=tmp_path, env=benv)
        assert r.returncode == 0, r.stdout + r.stderr
        assert r.stdout.splitlines() == [f"{n} -> {out.name}/{n[:-4]}{suffix}" for n in names] + ["process successfully done!"]
        assert f'"images": 4, "groups": {3 if budget else 1},' in r.stderr
        for n in names:
            assert (out / (n[:-4] + suffix)).read_bytes() == (tmp_path / "ref" / n).read_bytes(), n
