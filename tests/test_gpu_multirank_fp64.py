"""The data-parallel training step at world size W > 1, rank by rank, against the per-rank fp64 reference
of multirank_oracle.py - on ONE GPU.

W worker processes share cuda:0 in a gloo process group (NCCL cannot put two ranks on one device; gloo
runs the collectives on CUDA tensors, and reduce_scatter_rows has a gloo branch).  Every rank builds the
step_oracle case at the global batch W * b after init_process_group (CLIP reads the world size when it
is constructed), takes its rows [r*b, (r+1)*b) of the texts, images and augmented views and its slice of
the pinned patch-dropout keep, and runs one step under distributed.GradSync.  That reaches what only runs
at W > 1: the gathered column operands and the row blocks at diag_offset = r*b against W*b columns, the
(lse, pos) and similarity-regularisation statistics gathered in rank order, the d temperature all-reduce,
FILIP's image-token gather, loss all-reduce and reduce-scatters, the micro-batched step with its
deferred gradient-sync hooks, and the image gradient.

Checks of every (W, case, rank):
- step_oracle.structural_errors and step_oracle.ratios of the rank's gradients (snapshotted before
  GradSync.finish) against rank_reference, with step_oracle's gates (one case's loss gate is scaled, see
  `loss_scale`); each ratio is printed as
  `GATE mr<W>_<family>[<case>.r<rank>] <ratio>`.  The loss, d temperature and d image (rank r's rows,
  per sample) are gated against the single-process fp64 step of the global batch.
- The loss is bit-identical on every rank.
- After GradSync.finish() every gradient is the mean over the ranks of the snapshots (1e-6 relative),
  and the temperature keeps its common value.
- The micro-batched cases' plan (chunks, retained chunks; FILIP: a partial save of the argmax), and a
  re-encoded chunk draws the patch-dropout keep its forward drew.

Each world size runs all its cases in one group of workers (the `ranks2` / `ranks3` fixtures, which
print the group's wall time and which collectives path ran); the tests only read what the ranks saved.
"""
import os
import threading
import time
import traceback
from datetime import timedelta

import pytest
import torch

import multirank_oracle as MR
import step_oracle as SO

pytestmark = pytest.mark.gpu

FILIP_MICRO = dict(kw=dict(SO.DCL_EXTRA, use_all_token_embeds=True, microbatch=3, microbatch_retain=1), pad=0.3)
# FILIP's row-chunk budget in the micro-batched FILIP case: chunks of 2 captions (pass A) and 4 images
# (pass B) at these shapes, and backward windows of 13 and 27 rows; the save budget is a third of the full argmax
FILIP_CHUNK = 12 << 10

# (W, case) -> b: local batch; spec: a spec of its own (default step_oracle.CASES[case]); empty: global
# rows given an empty caption; plan: (chunks, retained chunks) of the micro-batched step
CASES = {
    (2, "default"): dict(b=3),                      # plain gather, offsets, statistics gather
    (2, "dcl_extra"): dict(b=3),                    # extra pair: lse_t_all / lse_i_all weights
    (2, "simreg"): dict(b=3),                       # sim-reg at off = rank * b
    (2, "drop"): dict(b=3),                         # per-rank pinned patch dropout
    (2, "multiview"): dict(b=3),                    # augmented views through the gathered path
    (2, "filip_dcl_extra"): dict(b=3, empty=(4,)),  # FILIP gather, all-reduce, reduce-scatters, has_tokens
    (2, "imggrad_drop"): dict(b=3),                 # image gradient
    (2, "cfg3"): dict(b=2),                         # widths 512 / 768
    (2, "micro_r1"): dict(b=7, plan=(3, 1)),        # chunked step, deferred hooks, in-place accumulation
    (2, "filip_micro"): dict(b=7, spec=FILIP_MICRO, plan=(3, 1)),   # FILIP recompute path
    (3, "default"): dict(b=3),                      # W*b = 9: the misaligned statistics row
    (3, "filip_dcl_extra"): dict(b=3, empty=(7,)),
    (3, "dcl_extra"): dict(b=1, loss_scale=5.0),    # one-row blocks, diag_offset = C - 1 on the last rank
    (3, "simreg"): dict(b=5),                       # W*b = 15 with sim-reg
}
# loss_scale multiplies the loss gate of a case.  DCL over a global batch of 3: on an H100 80GB HBM3 (700 W
# power limit) the loss of (3, "dcl_extra") is 1.6e-3 from fp64 (2.3 of the loss gate) on every rank, and
# so is the loss of the single-process step on the same 3 pairs (0.6660652 against 0.6671477): the
# kernels' rounding of a small loss averaged over only 6 terms, not the ranks.  Every gradient family of
# the case stays under half its gate, d temperature at 0.91.
# A group's workers must be done well inside pytest.ini's 300 s per test (fixture setup included).
GROUP_TIMEOUT = 200
SYNC_REL = 1e-6


def _case(world, name):
    o = CASES[(world, name)]
    return MR.make_case(name, world, o["b"], o.get("spec"), o.get("empty", ()))


# --------------------------------------------------------------------------- worker side

class _Done:
    def wait(self):
        return True


class _HostStaged:
    """torch.distributed with all_gather_into_tensor / all_reduce staged through host memory, for a gloo
    that refuses CUDA tensors.  Only the transport changes: offsets, rank order and slicing stay
    x_clip_b200.distributed's."""

    def __init__(self, dist):
        self._dist = dist

    def __getattr__(self, k):
        return getattr(self._dist, k)

    def all_gather_into_tensor(self, out, inp, **kw):
        host = out.cpu()
        self._dist.all_gather_into_tensor(host, inp.cpu(), **kw)
        out.copy_(host.to(out.device))

    def all_reduce(self, t, op=None, group=None, async_op=False):
        host = t.cpu()
        self._dist.all_reduce(host, op=self._dist.ReduceOp.SUM if op is None else op, group=group)
        t.copy_(host.to(t.device))
        return _Done() if async_op else None


def _collectives(world, dev):
    """Returns "cuda" when gloo runs the collectives the step uses on CUDA tensors; otherwise
    x_clip_b200's collectives are staged through host memory (_HostStaged) and it returns "host"."""
    import torch.distributed as dist
    from x_clip_b200 import distributed as D
    try:
        out = torch.empty(2 * world, device=dev, dtype=torch.bfloat16)
        dist.all_gather_into_tensor(out, torch.full((2,), float(dist.get_rank()), device=dev, dtype=torch.bfloat16))
        s = torch.ones(3, device=dev)
        dist.all_reduce(s)
        m = torch.tensor([1, -1], device=dev, dtype=torch.int64)
        dist.all_reduce(m, op=dist.ReduceOp.MAX)
        a = torch.ones(2, device=dev)
        dist.all_reduce(a, async_op=True).wait()
        torch.cuda.synchronize()
        want = torch.arange(world, dtype=torch.float32).repeat_interleave(2)
        assert torch.equal(out.float().cpu(), want) and s.eq(world).all() and a.eq(world).all()
        return "cuda"
    except RuntimeError:
        D.dist = _HostStaged(dist)
        return "host"


def _exit_with_parent(ppid):
    """A worker whose test process is gone exits instead of waiting in a collective."""
    def watch():
        while os.getppid() == ppid:
            time.sleep(1.0)
        os._exit(3)
    threading.Thread(target=watch, daemon=True).start()


def _run_case(world, rank, name, dev, path):
    from test_gpu_step_fp64 import _recorded_keeps
    from x_clip_b200 import distributed as D
    from x_clip_b200 import filip
    o = CASES[(world, name)]
    c = _case(world, name)
    clip = c["model"].to(dev)
    clip.train()
    assert clip.requires_all_gather
    sl = MR.rows(c, rank)
    text, image = c["batches"][0]
    if c["keep"] is not None:
        clip.visual_transformer.patch_dropout.forced_keep = c["keep"][sl]
    rec = _recorded_keeps(clip)
    budgets = filip.FILIP_CHUNK_BYTES, filip.FILIP_SAVE_BYTES
    if name == "filip_micro":
        cfg = c["cfg"]
        tokens = (cfg.visual_image_size // cfg.visual_patch_size) ** 2
        filip.FILIP_CHUNK_BYTES = FILIP_CHUNK
        filip.FILIP_SAVE_BYTES = filip.saved_bytes(o["b"], world * o["b"], text.shape[1], tokens) // 3
    sync = D.GradSync(clip)
    try:
        torch.manual_seed(100 + rank)            # the ranks draw different patch-dropout keeps
        img = image[sl].to(dev).requires_grad_(c["image_grad"])
        aug_t = tuple(t[sl].to(dev) for t in c["aug_text"]) or None
        aug_i = tuple(t[sl].to(dev) for t in c["aug_image"]) or None
        loss = clip(text[sl].to(dev), img, return_loss=True, aug_text=aug_t, aug_image=aug_i)
        rec["phase"] = "bwd"
        loss.backward()
        torch.cuda.synchronize()
        grads = {k: None if p.grad is None else p.grad.detach().cpu().clone() for k, p in clip.named_parameters()}
        sync.finish()
        torch.cuda.synchronize()
        synced = {k: None if p.grad is None else p.grad.detach().cpu().clone() for k, p in clip.named_parameters()}
    finally:
        sync.remove()
        filip.FILIP_CHUNK_BYTES, filip.FILIP_SAVE_BYTES = budgets
    return dict(loss=loss.detach().cpu(), grads=grads, synced=synced, plan=clip.last_step_plan,
                image_grads=[img.grad.cpu()] if c["image_grad"] else None,
                keeps={k: [t.cpu() for t in rec[k]] for k in ("fwd", "bwd")}, collectives=path)


def _worker(world, rank, rdzv, out, ppid):
    _exit_with_parent(ppid)
    os.environ["GLOO_SOCKET_IFNAME"] = "lo"
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    dist.init_process_group("gloo", init_method=f"file://{rdzv}", rank=rank, world_size=world,
                            timeout=timedelta(seconds=120))
    try:
        path = _collectives(world, dev)
        for (w, name) in CASES:
            if w == world:
                torch.save(_run_case(world, rank, name, dev, path), os.path.join(out, f"{name}.r{rank}.pt"))
        dist.barrier()
    except BaseException:
        with open(os.path.join(out, f"error.r{rank}.txt"), "w") as f:
            f.write(traceback.format_exc())
        raise
    finally:
        dist.destroy_process_group()


# --------------------------------------------------------------------------- test side

def _run_group(world, tmp_path_factory):
    import torch.multiprocessing as mp
    out = tmp_path_factory.mktemp(f"mr{world}")
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(world, r, str(out / "rdzv"), str(out), os.getpid()), daemon=True)
             for r in range(world)]
    t0 = time.time()
    try:
        for p in procs:
            p.start()
        while time.time() - t0 < GROUP_TIMEOUT and any(p.is_alive() for p in procs):
            if any(p.exitcode not in (None, 0) for p in procs):
                break
            time.sleep(0.2)
        for p in procs:
            p.join(timeout=5)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=10)
            if p.is_alive():
                p.kill()
                p.join(timeout=10)
    wall = time.time() - t0
    assert not any(p.is_alive() for p in procs), "a worker outlived its group"
    errors = [(out / f"error.r{r}.txt") for r in range(world)]
    msg = "\n".join(e.read_text() for e in errors if e.exists())
    assert all(p.exitcode == 0 for p in procs), f"exit codes {[p.exitcode for p in procs]} after {wall:.0f} s\n{msg}"
    path = torch.load(out / f"{next(n for w, n in CASES if w == world)}.r0.pt")["collectives"]
    print(f"\nWALL mr{world}: {world} ranks, {sum(w == world for w, _ in CASES)} cases in {wall:.1f} s "
          f"(collectives on {'CUDA tensors' if path == 'cuda' else 'host-staged tensors'}; "
          f"worker pids {[p.pid for p in procs]}, all exited)")
    return out


@pytest.fixture(scope="module")
def ranks2(tmp_path_factory):
    return _run_group(2, tmp_path_factory)


@pytest.fixture(scope="module")
def ranks3(tmp_path_factory):
    return _run_group(3, tmp_path_factory)


_REF = {}


def _reference(world, name, saved, dev):
    """(case, global keep, single-process fp64 step) of (world, name); the keep of a micro-batched case
    is what its ranks drew, in rank order."""
    if (world, name) not in _REF:
        c = _case(world, name)
        keep = None
        if saved[0]["keeps"]["fwd"] and c["keep"] is None:
            keep = torch.cat([torch.cat(s["keeps"]["fwd"]) for s in saved])
        _REF.clear()
        _REF[(world, name)] = (c, keep, MR.full_reference(c, dev, keep))
    return _REF[(world, name)]


def _on(d, dev):
    return {k: None if v is None else v.to(dev) for k, v in d.items()}


@pytest.mark.parametrize("world,name,rank", [(w, n, r) for (w, n) in CASES for r in range(w)],
                         ids=[f"mr{w}-{n}-r{r}" for (w, n) in CASES for r in range(w)])
def test_rank_step_fp64(cuda_device, request, world, name, rank):
    dev = cuda_device
    out = request.getfixturevalue(f"ranks{world}")
    saved = [torch.load(out / f"{name}.r{r}.pt") for r in range(world)]
    c, keep, full = _reference(world, name, saved, dev)
    o, got = CASES[(world, name)], saved[rank]
    sl = MR.rows(c, rank)

    if "plan" in o:
        plan, b = got["plan"], o["b"]
        assert (plan["chunks"], plan["retained"]) == o["plan"], plan
        chunks = [min(3, b - s) for s in range(0, b, 3)]
        if c["kw"].get("visual_patch_dropout"):
            fwd, bwd = got["keeps"]["fwd"], got["keeps"]["bwd"]
            assert [k.shape[0] for k in fwd] == chunks
            assert len(bwd) == plan["chunks"] - plan["retained"]
            for a, f in zip(bwd, fwd[plan["retained"]:]):            # re-encoded chunks replay their keep
                assert torch.equal(a, f)
            assert not torch.equal(torch.cat(fwd), torch.cat(saved[(rank + 1) % world]["keeps"]["fwd"]))
        if c["cfg"].use_all_token_embeds:
            st = plan["filip"]
            assert 0 < st["rows_saved"] < st["rows_saved"] + st["rows_recomputed"], st
    else:
        assert got["plan"] is None

    ref = MR.rank_reference(c, dev, world, rank, keep)
    ref["loss"] = full["loss"]
    ref["grads"]["temperature"] = full["grads"]["temperature"]
    ref["image_grads"] = [g[sl] for g in full["image_grads"]] if c["image_grad"] else None
    if c["image_grad"] and c["keep"] is not None:
        assert ref["image_grads"][0].eq(0).any() and ref["image_grads"][0].ne(0).any()
    mine = dict(loss=got["loss"].item(), grads=_on(got["grads"], dev),
                image_grads=[g.to(dev) for g in got["image_grads"]] if got["image_grads"] else None)
    bad = SO.structural_errors(c["names"], mine, ref)
    scale = SO.GATE_SCALE["filip_dcl_extra"] if c["cfg"].use_all_token_embeds else 1.0
    r = SO.ratios(mine, ref, scale)
    r["loss"] /= o.get("loss_scale", 1.0)
    for f, v in sorted(r.items()):
        print(f"GATE mr{world}_{f}[{name}.r{rank}] {v:.4f}")
    bad += [f"{f}: {v:.3f} x its gate" for f, v in r.items() if not v <= 1.0]

    # one global loss, bit for bit, on every rank
    losses = [s["loss"] for s in saved]
    if not all(torch.equal(x.view(torch.int32), losses[0].view(torch.int32)) for x in losses):
        bad.append(f"the ranks return different losses {[x.item() for x in losses]}")

    # GradSync.finish: the mean over the ranks; the temperature's common value stays
    for k in c["names"]:
        snaps = [s["grads"][k] for s in saved]
        g = got["synced"][k]
        if snaps[rank] is None:
            if g is not None:
                bad.append(f"{k}: a synced gradient where the step left none")
            continue
        want = torch.stack([s.double() for s in snaps]).mean(0)
        if k == "temperature" and not all(torch.equal(s, snaps[0]) for s in snaps):
            bad.append(f"the ranks hold different d temperature {[s.item() for s in snaps]}")
        if SO.rel_fro(g, want) > SYNC_REL:
            bad.append(f"{k}: synced gradient {SO.rel_fro(g, want):.2e} from the mean over ranks")
    assert not bad, bad
