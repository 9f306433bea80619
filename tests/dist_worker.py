"""One rank of the record exchange, for every world size from 1 up (tests/test_multigpu_gpu.py starts it; BASELINE.json
config 3, SURVEY.md 8(d)/(e)).  Each call shards world * B frames over the ranks in contiguous blocks
(smap_b200.dist.shard_range), every rank runs the whole path on its block and ONE ncclAllGather exchanges the records.

Every call has its own frames and scale rows, and each gathered block is compared byte for byte with the stage-wise
reference of THAT call for all world * B frames (tests/path_check.py: a second handle per rank that never runs the
whole path and has no communicator, so it is the 1-GPU result).  A call that read the other rec_buf, a stale
records_dev or the previous call's exchange returns a right-looking record and fails here.

What runs, at 96x160 unless stated:
  * the refusals: gather calls without a communicator (-52), rank / world out of range in smapb_comm_create and
    smapb_comm_attach (-1, before NCCL sees them, the handle's communicator and graphs untouched), B = 0;
  * smapb_infer_device_gather over eager, eager, capture and replays - plain, with do_flip, with RefineNet, with
    B < max_batch, and alternating with non-gather calls on the same pointers;
  * smapb_infer_device_gather_async with six calls outstanding before one smapb_gather_sync, three times: eager and
    captured calls in the first wave, replays after;
  * smapb_submit_host_gather on both slots alternately, with both batch sizes;
  * at 512x832 B = 8, bench.py's arrangement: two handles per rank, each with its own communicator and stream, both with
    batches in flight, in the deferred and in the host form; the same frames in batches of 4 on a third handle;
  * the communicator's life: init_comm twice, attach_torch_comm over an owned communicator, smapb_allgather_records over
    torch.distributed's communicator, and close() that leaves the borrowed communicator alive.
SMAPB_NCCL_EAGER=1 in the environment moves the all-gather out of the graph; the bytes, and so the digest, do not change.

At world = 1 the all-gather places nothing at a rank offset: every line above executes, but placement by rank is
checked only from two GPUs up (NCCL refuses two ranks on one device, so one GPU cannot stand in for two).  What is
pinned is which buffer goes where, not timing: a missing wait on gather_done would not reliably show, the exchange
takes microseconds and the forward milliseconds.

    RANK=0 WORLD_SIZE=1 LOCAL_RANK=0 MASTER_ADDR=127.0.0.1 MASTER_PORT=29511 python tests/dist_worker.py
    python -m torch.distributed.run --nproc-per-node 2 tests/dist_worker.py"""
import ctypes
import hashlib
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.join(HERE, "golden"), HERE, os.path.dirname(HERE)):
    sys.path.insert(0, p)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

MB = 3  # max_batch of the small handles


def main():
    import path_check
    from cases import refine_state_dict
    from smap_b200 import dist as sdist
    from smap_b200 import schema
    from smap_b200.engine import RECORD_BYTES, RECORD_DTYPE, Engine, SmapB200Error

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    sd = schema.make_state_dict(0, "identity")
    sha = hashlib.sha256()
    stats = dict(blocks=0, frames=0, persons=0)

    def engine(B, h, w, stream=None, refine=False):
        e = Engine(local, max_batch=B, in_h=h, in_w=w, stream=stream)
        e.load_state_dict(sd)
        if refine:
            e.load_refine_state_dict(refine_state_dict())
        return e

    def new_call(calls, B, flip=False, refine=False):
        """world * B frames of one call -> (this rank's frames and rows, the reference of all of them).  Every rank draws
        the same seeds in the same order, so all agree on what the call is."""
        parts = [calls.new(B, flip, refine) for _ in range(world)]
        lo, hi = sdist.shard_range(world * B, rank, world)
        assert (lo, hi) == (rank * B, rank * B + B)
        return parts[rank][0], parts[rank][1], torch.cat([p[2] for p in parts], 0)

    def check(got, want, what, gathered_block=True):
        """gathered_block: all world * B records of the call, the same bytes on every rank - only those enter the digest
        that the ranks compare at the end; a rank's own B records differ from its peers'."""
        got = got.cpu()
        assert torch.equal(got, want), "rank %d: %s differs from the stage-wise reference of its call" % (rank, what)
        if gathered_block:
            sha.update(got.numpy().tobytes())
        stats["blocks"] += 1
        stats["frames"] += got.shape[0]
        stats["persons"] += int(got.numpy().view(RECORD_DTYPE)["count"].sum())

    def refused(code, text, fn, *a, **kw):
        try:
            fn(*a, **kw)
        except SmapB200Error as e:
            assert "(%d)" % code in str(e) and text in str(e), e
            return
        raise AssertionError("accepted: expected %d (%s)" % (code, text))

    def zeros(n, pinned=False):
        t = torch.zeros(n, RECORD_BYTES, dtype=torch.uint8, device="cpu" if pinned else dev)
        return t.pin_memory() if pinned else t

    st = torch.cuda.Stream(dev)
    eng = engine(MB, path_check.H, path_check.W, st, refine=True)
    ref = engine(MB, path_check.H, path_check.W, refine=True)
    calls = path_check.Calls(ref)
    lib, h = eng.lib, eng._h
    xd = torch.zeros(MB, 3, path_check.H, path_check.W, device=dev)  # the pointers that graphs are captured on
    rows = torch.zeros(MB, 9, dtype=torch.float64, device=dev)

    def on_pointers(B, x, s):
        """The call's content copied into the captured tensors, and the handle's stream ordered after the copy."""
        xd[:B].copy_(x)
        rows[:B].copy_(s)
        st.wait_stream(torch.cuda.current_stream(dev))
        return xd[:B], rows[:B]

    def gathered(B, flip=False, refine=False, what="gather"):
        x, s, want = new_call(calls, B, flip, refine)
        out = zeros(world * B)
        x, s = on_pointers(B, x, s)
        eng.infer_device(x, s, do_flip=flip, out=out, gather=True)
        st.synchronize()
        check(out, want, what)

    def plain(B, what):
        x, s, want = new_call(calls, B)
        out = zeros(B)
        x, s = on_pointers(B, x, s)
        eng.infer_device(x, s, out=out)
        st.synchronize()
        check(out, want[rank * B:rank * B + B], what, gathered_block=False)

    # ---- refusals; each returns before any launch --------------------------------------------------------------------
    x, s, _ = new_call(calls, MB)
    x, s = on_pointers(MB, x, s)
    out = zeros(MB)  # a handle without a communicator takes itself for a world of one
    refused(-52, "no communicator", eng.infer_device, x, s, out=out, gather=True)
    refused(-52, "no communicator", eng.infer_device, x, s, out=out, gather=True, defer=True)
    refused(-52, "no communicator", eng.submit_host, 0, x.cpu().pin_memory(), s.cpu().pin_memory(), zeros(MB, True),
            gather=True)
    refused(-52, "no NCCL communicator", eng.allgather, zeros(MB))
    assert lib.smapb_allgather_records(h, None, ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(out.data_ptr()), 0, None) == -1
    assert b"B < 1" in lib.smapb_last_error(h)
    uid = (ctypes.c_char * 128)()
    for r, w in ((world, world), (-1, world), (0, 0), (0, -1)):  # never an in-range rank whose peers do not exist
        assert lib.smapb_comm_create(h, uid, r, w) == -1, (r, w)
        assert b"out of range" in lib.smapb_last_error(h)
    refused(-52, "no communicator", eng.infer_device, x, s, out=out, gather=True)  # still none

    # ---- one handle, its own communicator ------------------------------------------------------------------------------
    eng.init_comm()
    sdist.sync_tile_table()
    for i in range(5):  # eager, eager, capture, replay, replay
        gathered(MB, what="stream-ordered gather %d" % i)
    for i in range(4):
        gathered(MB, flip=True, what="gather with do_flip %d" % i)
    for i in range(4):
        gathered(1, what="gather of B=1 on a max_batch=3 handle %d" % i)
    for i in range(3):  # (3, no flip, no gather) has its two eager runs here and is captured on the gather graph's pointers
        plain(MB, "non-gather call %d" % i)
    for i in range(3):
        gathered(MB, what="gather alternating with non-gather %d" % i)
        plain(MB, "non-gather alternating with gather %d" % i)
    eng.set_refine(True)
    for i in range(4):
        gathered(MB, refine=True, what="gather with RefineNet %d" % i)
    eng.set_refine(False)
    gathered(MB, what="gather after set_refine(False)")
    plain(MB, "non-gather call after set_refine(False)")  # captured again: set_refine dropped every graph

    # deferred: six calls outstanding, each with its own tensors and its own output.  With do_flip, which no non-gather
    # call has used yet: the first two calls of wave 0 run eagerly and write rec_buf[0] and rec_buf[1] directly, while
    # records_dev still holds an earlier call's records; the other four are captured.  Wave 1 captures those two and
    # replays four, wave 2 replays all six.
    ins = [(torch.zeros_like(xd), torch.zeros_like(rows)) for _ in range(6)]
    for wave in range(3):
        wants, outs = [], []
        for xi, si in ins:
            x, s, want = new_call(calls, MB, flip=True)
            xi.copy_(x)
            si.copy_(s)
            wants.append(want)
            outs.append(zeros(world * MB))
        st.wait_stream(torch.cuda.current_stream(dev))
        for (xi, si), o in zip(ins, outs):
            eng.infer_device(xi, si, do_flip=True, out=o, gather=True, defer=True)
        eng.gather_sync()
        st.synchronize()
        for i, (o, want) in enumerate(zip(outs, wants)):
            check(o, want, "deferred exchange %d of wave %d" % (i, wave))

    # host form: H2D, path, device all-gather, ONE D2H; both slots, both batch sizes
    batches = []
    for i in range(6):
        B = MB if (i // 2) % 2 == 0 else 1
        x, s, want = new_call(calls, B)
        batches.append((x.pin_memory(), s.pin_memory(), zeros(world * B, True), want))
    for i, (x, s, o, _) in enumerate(batches):
        if i >= 2:
            eng.wait(i % 2)
        eng.submit_host(i % 2, x, s, o, gather=True)
    eng.wait(0)
    eng.wait(1)
    for i, (_, _, o, want) in enumerate(batches):
        check(o, want, "host gather %d (slot %d, B=%d)" % (i, i % 2, o.shape[0] // world))

    # ---- the communicator's life ---------------------------------------------------------------------------------------
    eng.init_comm()  # the first communicator is destroyed, gather graphs go, non-gather graphs stay
    plain(MB, "non-gather replay after a second init_comm")
    for i in range(4):
        gathered(MB, what="gather after a second init_comm %d" % i)
    pg = dist.distributed_c10d._get_default_group()._get_backend(dev)
    if not pg._is_initialized():
        pg.eager_connect_single_device(dev)
    torch_comm = ctypes.c_void_p(pg._comm_ptr())
    for r, w in ((world, world), (-1, world), (0, 0)):
        assert lib.smapb_comm_attach(h, torch_comm, r, w) == -1, (r, w)
        assert b"out of range" in lib.smapb_last_error(h)
    gathered(MB, what="gather replay after refused smapb_comm_attach calls")
    plain(MB, "non-gather replay after refused smapb_comm_attach calls")
    eng.attach_torch_comm()  # the owned communicator is replaced by a borrowed one
    for i in range(3):
        gathered(MB, what="gather over torch.distributed's communicator %d" % i)
    x, s, want = new_call(calls, MB)
    allr = eng.allgather(want[rank * MB:rank * MB + MB].to(dev))  # the exchange step alone
    st.synchronize()
    check(allr, want, "smapb_allgather_records over torch.distributed's communicator")
    eng.close()
    dist.barrier()  # close() left the borrowed communicator alive

    # ---- bench.py's arrangement at its shape: two handles per rank, own communicators, both with batches in flight ---------
    B, H, W = 8, 512, 832
    big_ref = engine(B, H, W)
    big_calls = path_check.Calls(big_ref, H, W, first_seed=1000)
    pair = [engine(B, H, W, torch.cuda.Stream(dev)) for _ in range(2)]
    for e in pair:  # the same order on every rank
        e.init_comm()
    work = []
    for i in range(6):
        x, s, want = new_call(big_calls, B)
        work.append((x.to(dev), s.to(dev), zeros(world * B), want))
    for e in pair:
        e.stream.wait_stream(torch.cuda.current_stream(dev))
    for i, (x, s, o, _) in enumerate(work):
        pair[i % 2].infer_device(x, s, out=o, gather=True, defer=True)
    for e in pair:
        e.gather_sync()
        e.stream.synchronize()
    for i, (_, _, o, want) in enumerate(work):
        check(o, want, "512x832 deferred exchange %d on handle %d" % (i, i % 2))
    host = [(x.cpu().pin_memory(), s.cpu().pin_memory(), zeros(world * B, True), want) for x, s, _, want in work[:4]]
    for i, (x, s, o, _) in enumerate(host):
        pair[i % 2].submit_host((i // 2) % 2, x, s, o, gather=True)
    for i in range(4):
        pair[i % 2].wait((i // 2) % 2)
    for i, (_, _, o, want) in enumerate(host):
        assert torch.equal(o, want), "rank %d: 512x832 host gather %d on handle %d" % (rank, i, i % 2)
    # the same frames in batches of 4 on the 1-GPU side (tile boundaries move, bits must not)
    half = engine(B // 2, H, W)
    x, s, _, want = work[0]
    mine = want[rank * B:rank * B + B]
    got = torch.cat([half.infer_device(x[k:k + B // 2], s[k:k + B // 2]).cpu() for k in (0, B // 2)], 0)
    assert torch.equal(got, mine), "batch split changed the records"
    for e in pair + [half, big_ref, ref]:
        e.close()

    # all ranks gathered the same bytes
    digest = torch.tensor([int.from_bytes(sha.digest()[:7], "little")], device=dev)
    alld = [torch.zeros_like(digest) for _ in range(world)]
    dist.all_gather(alld, digest)
    assert all(int(d) == int(digest) for d in alld)
    if rank == 0:
        print("EXCHANGE OK world=%d blocks=%d frames=%d persons=%d nccl_in_graph=%d sha=%s" % (
            world, stats["blocks"], stats["frames"], stats["persons"], "SMAPB_NCCL_EAGER" not in os.environ,
            sha.hexdigest()[:16]))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
