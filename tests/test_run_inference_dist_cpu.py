"""CPU: the host logic of run_inference's distributed mode (smap_b200.run_inference.run_distributed) over gloo.

 * step_plan: every frame is taken exactly once, by one rank at one step, and the real gathered slots of the steps, in
   order, are the frames 0 ... n-1;
 * drive(), the rank / step / reassembly loop, with records faked from each file's index and exchanged by gloo: rank 0
   appends the same (record, name) sequence at world 2 and 3 as at world 1, and the clamp counts add up over the ranks;
 * failure agreement: one rank raising in any stage of a step (or rank 0 failing to append) makes every rank raise and
   exit nonzero, promptly;
 * the CLI: without WORLD_SIZE main() calls run() exactly as before; with it, a missing checkpoint makes every rank
   return 1."""
import os
import socket
import subprocess
import sys
import time

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from smap_b200 import run_inference as R
from smap_b200._lib import RECORD_BYTES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("batch", [1, 2, 8])
def test_step_plan_takes_every_frame_once_in_slot_order(world, batch):
    for n in sorted({0, 1, world - 1, world, batch, world * batch - 1, world * batch, world * batch + 1, 3 * world * batch,
                     3 * world * batch + batch + 1, 37}):
        if n < 0:
            continue
        plan = R.step_plan(n, world, batch)
        assert len(plan) == -(-n // (world * batch))
        taken, real = [], []
        for s, (shards, slots) in enumerate(plan):
            assert len(shards) == world
            for r, f in enumerate(shards):
                assert len(f) <= batch
                assert list(f) == [i for i in range((s * world + r) * batch, (s * world + r + 1) * batch) if i < n]
                taken.extend(f)
            assert slots == sorted(slots) and all(0 <= k < world * batch for k in slots)
            # slot r * batch + k of the gathered block holds shards[r][k]
            real.extend(shards[k // batch][k % batch] for k in slots)
            if s < len(plan) - 1:
                assert slots == list(range(world * batch))
        assert sorted(taken) == list(range(n))
        assert real == list(range(n))


def _fake_record(i):
    return torch.from_numpy(np.random.default_rng(1000 + i).integers(0, 256, RECORD_BYTES, dtype=np.uint8))


class _FakeSteps:
    """drive()'s steps with the GPU replaced: a frame's record is drawn from the index written in its file, the exchange
    is dist.allgather_records over gloo, and its clamp count is index + 1; padded slots stay zero.  fail = (stage, rank,
    step) raises there."""

    def __init__(self, paths, batch, fail=None):
        import torch.distributed as dist

        self.paths, self.batch, self.fail, self.step = paths, batch, fail, -1
        self.rank, self.sat = dist.get_rank(), 0

    def _maybe_fail(self, stage):
        if self.fail and self.fail[0] == stage and self.fail[1] == self.rank and self.fail[2] == self.step:
            raise RuntimeError("injected %s failure on rank %d" % (stage, self.rank))

    def prepare(self, frames):
        self.step += 1
        self._maybe_fail("prepare")
        self.local = torch.zeros(self.batch, RECORD_BYTES, dtype=torch.uint8)
        for k, i in enumerate(frames):
            with open(self.paths[i]) as f:
                idx = int(f.read())
            self.local[k] = _fake_record(idx)
            self.sat += idx + 1

    def submit(self):
        self._maybe_fail("submit")

    def collect(self):
        """The exchange runs here, once every rank has submitted (the GPU's is enqueued by submit and waited for here)."""
        from smap_b200 import dist as sdist

        out = sdist.allgather_records(self.local)
        self._maybe_fail("collect")
        return out

    def saturation(self):
        return self.sat


def _make_dir(root, n):
    """n files in nested directories; the index written in each is its position in list_images' order."""
    names = ["d%d/%s%02d.%s" % (i % 3, "ab"[i % 2], i, ("jpg", "png", "jpeg")[i % 3]) for i in range(n)]
    for name in names:
        os.makedirs(os.path.dirname(os.path.join(root, name)), exist_ok=True)
        open(os.path.join(root, name), "w").close()
    paths = R.list_images(root)
    for i, p in enumerate(paths):
        with open(p, "w") as f:
            f.write(str(i))
    return paths


def _drive_worker(rank, world, port, root, batch, fail, q):
    import torch.distributed as dist

    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    seq = []
    rc = 0
    try:
        box = [R.list_images(root) if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        paths = box[0]

        def append(rec, frames):
            assert rec.shape == (len(frames), RECORD_BYTES)
            if fail and fail[0] == "append" and len(seq) >= fail[2] * world * batch:
                raise OSError("injected append failure")
            seq.extend((bytes(r.numpy()), R.image_name(paths[i], root)) for r, i in zip(rec, frames))

        sat = R.drive(len(paths), batch, _FakeSteps(paths, batch, fail), append)
        q.put((rank, "ok", seq if rank == 0 else None, sat))
    except R.RankFailed as e:
        q.put((rank, "RankFailed", e.pending, None))
        rc = 1
    except Exception as e:
        q.put((rank, type(e).__name__, str(e), None))
        rc = 1
    finally:
        dist.destroy_process_group()
    sys.exit(rc)


def _run_ranks(world, root, batch, fail=None, timeout=120):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _port()
    procs = [ctx.Process(target=_drive_worker, args=(r, world, port, root, batch, fail, q)) for r in range(world)]
    t0 = time.monotonic()
    for p in procs:
        p.start()
    try:
        got = {}
        for _ in range(world):
            r, *rest = q.get(timeout=timeout)
            got[r] = rest
        for p in procs:
            p.join(timeout=max(1.0, timeout - (time.monotonic() - t0)))
    finally:
        alive = [p for p in procs if p.is_alive()]
        for p in alive:
            p.kill()
            p.join()
    assert not alive, "ranks still running after %d s" % timeout
    return got, [p.exitcode for p in procs], time.monotonic() - t0


@pytest.mark.parametrize("n,batch", [(23, 4), (16, 4), (5, 8), (0, 2)])
def test_drive_at_world_2_and_3_appends_the_one_process_sequence(tmp_path, n, batch):
    paths = _make_dir(str(tmp_path), n)
    want = [(bytes(_fake_record(i).numpy()), R.image_name(p, str(tmp_path))) for i, p in enumerate(paths)]
    ref, codes, _ = _run_ranks(1, str(tmp_path), batch)
    assert codes == [0] and ref[0][0] == "ok"
    assert ref[0][1] == want
    assert ref[0][2] == n * (n + 1) // 2
    for world in (2, 3):
        got, codes, _ = _run_ranks(world, str(tmp_path), batch)
        assert codes == [0] * world, got
        assert got[0][1] == want, "world %d: rank 0 appended another sequence" % world
        assert all(got[r][2] == n * (n + 1) // 2 for r in range(world)), "clamp counts do not add up over the ranks"


@pytest.mark.parametrize("stage,rank,step", [("prepare", 1, 0), ("submit", 1, 1), ("collect", 0, 2), ("append", 0, 1),
                                             ("prepare", 2, 3)])
def test_a_failing_rank_stops_every_rank(tmp_path, stage, rank, step):
    """3 ranks, batch 2, 19 frames: 4 steps, the last one ragged (rank 2 has no frame in it)."""
    _make_dir(str(tmp_path), 19)
    got, codes, secs = _run_ranks(3, str(tmp_path), 2, fail=(stage, rank, step), timeout=60)
    assert all(c == 1 for c in codes), (codes, got)
    assert secs < 60
    for r in range(3):
        if r == rank:
            assert got[r][0] == ("OSError" if stage == "append" else "RuntimeError"), got[r]
        else:
            assert got[r][0] == "RankFailed", got[r]
            # only a failed submission leaves the others' exchange of that step waiting for it
            assert got[r][1] == (stage == "submit"), got[r]


def test_plain_cli_calls_run_as_before(tmp_path, monkeypatch, capsys):
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    torch.save({"model": {"w": torch.zeros(1)}}, tmp_path / "smap.pth")
    calls = []

    def fake_run(*a, **kw):
        calls.append((a, kw))
        kw["stats"]["saturation"] = 7
        return 3

    def no_dist(*a, **kw):
        raise AssertionError("the distributed driver ran without WORLD_SIZE")

    monkeypatch.setattr(R, "run", fake_run)
    monkeypatch.setattr(R, "run_distributed", no_dist)
    out_dir = tmp_path / "out"
    rc = R.main(["-p", str(tmp_path / "smap.pth"), "--dataset_path", str(tmp_path), "--batch_size", "4", "--do_flip", "1",
                 "--json_name", "x", "--output_dir", str(out_dir), "--precision", "fp16", "--glob_order", "1"])
    assert rc == 0
    (a, kw), = calls
    out = str(out_dir / "stage3_root2_run_inference_test_x.json")
    assert a[1:] == (str(tmp_path), out, None, 4, 1.0, "CMU")
    assert set(a[0]) == {"w"}
    assert kw == dict(glob_order=True, precision="fp16", stats={"saturation": 7}, jpeg_colour=False)
    text = capsys.readouterr().out
    assert "Pairs writed to {} (3 images)".format(out) in text
    assert "fp16: 7 activation values exceeded +-65504" in text
    assert out_dir.is_dir()
    monkeypatch.setattr(R, "run", no_dist)
    assert R.main(["-p", str(tmp_path / "missing.pth"), "-rp", str(tmp_path / "r.pth")]) == 1
    assert capsys.readouterr().out.strip() == "No such checkpoint of SMAP " + str(tmp_path / "missing.pth")
    assert R.main(["-p", str(tmp_path / "smap.pth"), "-rp", str(tmp_path / "r.pth"), "--dataset_path", str(tmp_path)]) == 1
    assert capsys.readouterr().out.strip() == "No such RefineNet checkpoint of " + str(tmp_path / "r.pth")


def test_cli_under_torchrun_variables_stops_every_rank_on_a_missing_checkpoint(tmp_path):
    port = _port()
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, "-m", "smap_b200.run_inference", "-p", str(tmp_path / "none.pth"),
                                       "--dataset_path", str(tmp_path), "--output_dir", str(tmp_path / "out")],
                                      cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    try:
        outs = [p.communicate(timeout=120)[0] for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    assert [p.returncode for p in procs] == [1, 1], outs
    for rank, text in enumerate(outs):
        assert "rank %d: No such checkpoint of SMAP" % rank in text, text
        assert "Pairs writed" not in text
