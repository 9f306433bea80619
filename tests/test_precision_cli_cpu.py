"""CPU: the --precision option of the run_inference driver reaches the engine, and an unknown precision is rejected."""
import pytest
import torch

from smap_b200 import run_inference as R
from smap_b200.engine import PRECISIONS


def test_precisions_offered():
    assert set(PRECISIONS) == {"bf16x3", "fp16", "bf16"}


@pytest.mark.parametrize("precision", [None, "bf16x3", "fp16", "bf16"])
def test_cli_passes_the_precision_through(tmp_path, monkeypatch, capsys, precision):
    ckpt = tmp_path / "SMAP.pth"
    torch.save({"model": {}}, str(ckpt))
    got = {}

    def fake_run(*args, **kw):
        got.update(kw)
        kw["stats"]["saturation"] = 7 if kw["precision"] == "fp16" else 0
        return 0

    monkeypatch.setattr(R, "run", fake_run)
    argv = ["-p", str(ckpt), "--dataset_path", str(tmp_path), "--output_dir", str(tmp_path / "out")]
    if precision:
        argv += ["--precision", precision]
    assert R.main(argv) == 0
    assert got["precision"] == (precision or "bf16x3")  # the default stays the parity mode
    out = capsys.readouterr().out
    assert ("7 activation values exceeded" in out) == (precision == "fp16")


def test_cli_rejects_an_unknown_precision(tmp_path, capsys):
    with pytest.raises(SystemExit) as e:
        R.main(["-p", str(tmp_path / "x.pth"), "--precision", "fp8"])
    assert e.value.code == 2
    assert "invalid choice: 'fp8'" in capsys.readouterr().err


def test_run_rejects_an_unknown_precision_before_touching_the_gpu(tmp_path):
    with pytest.raises(ValueError, match="unknown precision 'tf32'"):
        R.run({}, str(tmp_path), str(tmp_path / "o.json"), precision="tf32")
