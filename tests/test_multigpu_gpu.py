"""GPU: sharding invariance (BASELINE.json config 3, SURVEY.md 8(d)/(e) "result independent of G").

 * one GPU: the records of 16 frames do not depend on how the frames are split into batches (8+8, 4x4, 16x1 ...) nor on the
   handle - the compute half of the invariance;
 * the exchange: tests/dist_worker.py, one process per rank.  At world = 1 on every machine: NCCL makes a communicator of
   one rank, so every line of the exchange code runs (the in-graph all-gather, the deferred exchange on the gather
   stream, the host form, the communicator's life cycle) and what is gathered must equal the stage-wise reference of
   each call.  Once more with SMAPB_NCCL_EAGER=1 (the all-gather behind the graph instead of inside it) and with
   SMAPB_NCCL_LIB naming a file that does not exist (the library's own fall-back names must still load NCCL): the same
   digest.  At world = 2 or 8 where the machine has the GPUs - only there is the placement of a rank's records at its
   offset checked, because NCCL refuses two ranks on one device."""
import os
import re
import signal
import socket
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from smap_b200 import schema

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_records_do_not_depend_on_batch_split_or_handle():
    from smap_b200.engine import Engine, scale_row

    sd = schema.make_state_dict(0, "identity")
    total = 16
    frames = torch.cat([schema.make_input(1, 512, 832, seed=2000 + i) for i in range(total)], 0).cuda()
    sc = dict(scale=832 / 1920, img_width=1920, img_height=1080, net_width=832, net_height=512, f_x=1920.0, f_y=1920.0,
              cx=960.0, cy=540.0)
    row = scale_row(sc)
    results = {}
    for B in (8, 4, 1):
        e = Engine(0, max_batch=B, in_h=512, in_w=832)
        e.load_state_dict(sd)
        scales = torch.from_numpy(np.stack([row] * B)).cuda()
        # 3 passes over the first block exercise eager run -> graph capture -> replay as well
        for _ in range(3):
            first = e.infer_device(frames[:B], scales).cpu()
        rec = torch.cat([e.infer_device(frames[k:k + B], scales).cpu() for k in range(0, total, B)], 0)
        assert torch.equal(rec[:B], first)
        results[B] = rec
        e.close()
    assert torch.equal(results[8], results[4]), "8-frame vs 4-frame batches"
    assert torch.equal(results[8], results[1]), "8-frame vs single-frame batches"


def run_worker(world, tmp_path, extra_env=None, timeout=600):
    """Start tests/dist_worker.py once per rank, each in a session of its own, and return what rank 0 reported once all
    have ended.  As soon as one rank fails, or at the timeout, every rank's whole process group is killed: its peers
    would otherwise wait for it in a collective."""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs, logs = [], []
    try:
        for rank in range(world):
            env = dict(os.environ, RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                       MASTER_PORT=str(port), **(extra_env or {}))
            logs.append(open(tmp_path / ("rank%d.log" % rank), "w+"))
            procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "dist_worker.py")], cwd=ROOT, env=env,
                                          stdout=logs[-1], stderr=subprocess.STDOUT, start_new_session=True))
        deadline = time.monotonic() + timeout
        while True:
            codes = [p.poll() for p in procs]
            if all(c is not None for c in codes) or any(c for c in codes) or time.monotonic() > deadline:
                break
            time.sleep(0.2)
    finally:
        for p in procs:
            try:
                os.killpg(p.pid, signal.SIGKILL)
            except ProcessLookupError:
                pass
            p.wait()
        texts = []
        for f in logs:
            f.seek(0)
            texts.append(f.read())
            f.close()
    assert None not in codes or any(codes), "no result after %d s" % timeout
    assert codes == [0] * world, "\n".join("--- rank %d (exit %s)\n%s" % (r, c, x[-4000:]) for r, (c, x) in enumerate(zip(codes, texts)))
    m = re.search(r"EXCHANGE OK world=%d blocks=(\d+) frames=\d+ persons=(\d+) nccl_in_graph=(\d) sha=(\w+)" % world, texts[0])
    assert m, texts[0][-2000:]
    print("\n" + m.group(0))
    assert int(m.group(1)) > 50 and int(m.group(2)) > 0
    return int(m.group(3)), m.group(4)


def test_exchange_on_one_gpu_equals_the_stagewise_reference_in_graph_and_eager(tmp_path):
    in_graph, sha = run_worker(1, tmp_path)
    assert in_graph == 1
    (tmp_path / "eager").mkdir()
    in_graph, sha_eager = run_worker(1, tmp_path / "eager", {"SMAPB_NCCL_EAGER": "1",
                                                             "SMAPB_NCCL_LIB": str(tmp_path / "no_such_libnccl.so")})
    assert in_graph == 0
    assert sha_eager == sha, "with SMAPB_NCCL_EAGER=1 (and SMAPB_NCCL_LIB naming a missing file) other bytes were gathered"


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="placement by rank needs >= 2 GPUs")
def test_sharded_allgather_equals_single_gpu_result(tmp_path):
    world = 8 if torch.cuda.device_count() >= 8 else 2
    run_worker(world, tmp_path, timeout=900)
