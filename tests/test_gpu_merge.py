"""The multi-GPU TSDF merge (`gsb_tsdf_reduce`, csrc/gsb_reduce.cu) bit for bit against its host restatement
(tests/merge_oracle.py), with 2 and 3 ranks, as an all-reduce, a reduce to rank 0 (the canonical rank exchanges its pool in
place) and a reduce to the last rank, with and without colour.

The ranks are separate processes (tests/merge_ranks.py) started here and joined through an NCCL id in a file:
  * one_gpu: every rank on device 0.  Each rank gets its own NCCL_HOSTID, so NCCL takes the ranks for separate nodes
    (instead of refusing a duplicate GPU) and moves the data through its socket transport on the loopback interface.
  * per_gpu: rank r on device r, where the machine has enough devices.
Bars: with 2 ranks every element bit for bit and the merge's drop count exact; with 3 ranks every element one of the
values NCCL's choice of summation order (or a reduction in extra precision) gives, and the drop count within its bounds."""
import os
import socket
import subprocess
import sys
import time

import numpy as np
import pytest

from tests import merge_ranks as MR
from tests.merge_oracle import check_rank, merge_oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GSB_ERR_WORKSPACE = 2
LAUNCH_TIMEOUT_S = 300


class Launch:
    def __init__(self, world, out_dir, seconds):
        self.world, self.dir, self.seconds = world, out_dir, seconds

    def rec(self, cid, rank):
        with np.load(os.path.join(self.dir, f"{cid}_r{rank}.npz")) as z:
            return {k: z[k] for k in z.files}


def _free_port():
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _tail(path, n=4000):
    try:
        with open(path, errors="replace") as fh:
            return fh.read()[-n:]
    except OSError:
        return ""


def _launch(mode, world, out_dir):
    """Runs `world` rank processes to the end of the case list; returns a Launch, or raises / skips with every rank's
    stderr.  No child outlives this call."""
    import torch

    if mode == "per_gpu" and torch.cuda.device_count() < world:
        pytest.skip(f"per_gpu needs {world} CUDA devices, this machine has {torch.cuda.device_count()}")
    port = _free_port()
    procs, logs = [], []
    t0 = time.monotonic()
    try:
        for r in range(world):
            env = dict(os.environ, NCCL_SOCKET_IFNAME="lo", NCCL_IB_DISABLE="1", MASTER_ADDR="127.0.0.1")
            if mode == "one_gpu":
                env["NCCL_HOSTID"] = f"gsbtest{r}"
            log = os.path.join(out_dir, f"rank{r}.log")
            logs.append(log)
            cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
                "-m", "tests.merge_ranks", "--rank", str(r), "--world", str(world), "--mode", mode, "--dir", str(out_dir),
                "--port", str(port)]
            with open(log, "w") as fh:
                procs.append(subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=fh, stderr=subprocess.STDOUT))
        deadline = t0 + LAUNCH_TIMEOUT_S
        while any(p.poll() is None for p in procs) and time.monotonic() < deadline:
            if any(p.poll() not in (None, 0) for p in procs):
                time.sleep(2.0)  # let the others report too, then stop them
                break
            time.sleep(0.2)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        for p in procs:
            p.wait()
    codes = [p.returncode for p in procs]
    refused = [_tail(os.path.join(out_dir, f"refused_r{r}.txt")) for r in range(world)]
    if any(refused):
        msg = next(m for m in refused if m)
        if mode == "one_gpu":
            pytest.skip(f"NCCL refused {world} ranks on one device with distinct NCCL_HOSTID: {msg}")
        raise AssertionError(f"gsb_comm_create failed: {msg}")
    if codes != [0] * world:
        raise AssertionError(f"rank exit codes {codes} after {time.monotonic() - t0:.0f} s (limit {LAUNCH_TIMEOUT_S} s):\n" +
                             "\n".join(f"--- rank {r} ---\n{_tail(logs[r])}" for r in range(world)))
    return Launch(world, str(out_dir), time.monotonic() - t0)


@pytest.fixture(scope="module")
def launches(gsb_lib, cuda_device, tmp_path_factory):
    cache = {}

    def get(mode, world):
        if (mode, world) not in cache:
            try:
                cache[(mode, world)] = _launch(mode, world, tmp_path_factory.mktemp(f"merge_{mode}_{world}"))
            except BaseException as e:  # a skip or a failure is the same for every test of this launch
                cache[(mode, world)] = e
        got = cache[(mode, world)]
        if isinstance(got, BaseException):
            raise got
        return got

    return get


MODES = [pytest.param(m, w, id=f"{m}-{w}ranks") for m in ("one_gpu", "per_gpu") for w in (2, 3)]


# ----------------------------------------------------------------------------------------------------------- helpers

def _units(rec, prefix):
    keys = [tuple(int(v) for v in k) for k in rec[f"{prefix}_keys"]]
    tw = rec[f"{prefix}_tw"]
    col = rec.get(f"{prefix}_col")
    return {k: (tw[i], None if col is None else col[i]) for i, k in enumerate(keys)}


def _dead(rec):
    return {tuple(int(v) for v in k) for k in rec["pre_dead"]}


def _dst(root, world):
    r = MR.root_of(root, world)
    return None if r < 0 else r


def _check_merge(L, cid, root, prefix="call0", pool=None):
    """Every receiving rank's bricks after the merge against the oracle of all ranks' bricks before it; every other rank's
    volume unchanged bit for bit."""
    world = L.world
    recs = [L.rec(cid, r) for r in range(world)]
    dst = _dst(root, world)
    pool = int(recs[0]["pool"]) if pool is None else pool
    exp = merge_oracle([_units(x, "pre") for x in recs], dst, pool, [_dead(x) for x in recs])
    canon = 0 if dst is None else dst
    canon_keys = set(_units(recs[canon], prefix))
    for r in range(world):
        x = recs[r]
        if r in exp:
            got = _units(x, prefix)
            drops = int(x[f"{prefix}_stats"][1] - x["pre_stats"][1])
            check_rank(exp[r], got, drops, canon_keys, f"{cid} rank {r}")
            assert int(x[f"{prefix}_stats"][0]) == len(got)
        elif int(x[f"{prefix}_stats"][2]) == int(x["pre_stats"][2]):
            assert str(x[f"{prefix}_digest"]) == str(x["pre_digest"]), f"{cid}: rank {r} does not receive, yet its volume changed"
        else:  # grown to the ranks' largest pool before the merge: the same bricks, bit for bit, in a larger pool
            a, b = _units(x, prefix), _units(x, "pre")
            assert set(a) == set(b), f"{cid}: rank {r} does not receive, yet its bricks changed"
            for k in b:
                assert np.array_equal(a[k][0].view(np.uint32), b[k][0].view(np.uint32)), f"{cid}: rank {r} brick {k} changed"
                if b[k][1] is not None:
                    assert np.array_equal(a[k][1].view(np.uint32), b[k][1].view(np.uint32)), f"{cid}: rank {r} brick {k} changed"
    return recs, exp


def _run_all(checks):
    """Runs every check, then fails with all the failures at once."""
    errors = []
    for what, fn in checks:
        try:
            fn()
        except AssertionError as e:
            errors.append(f"{what}: {e}")
    assert not errors, f"{len(errors)} of {len(checks)} cases failed:\n" + "\n".join(errors)


# ----------------------------------------------------------------------------------------------------------- tests

PLAIN = ("disjoint", "identical", "partial", "one_empty", "all_empty", "collide", "fill_exact", "overflow", "pre_overflow",
         "alpha")


@pytest.mark.parametrize("mode,world", MODES)
def test_merge_matches_host_restatement(launches, mode, world):
    """Disjoint, identical and partly overlapping brick sets (rank 1 opens its bricks in reverse order, so the canonical
    order is not its pool order), an empty rank, all ranks empty, keys that share home slots at the ends of the lattice,
    a union that fills the pool exactly, one that exceeds it by 3, a rank whose own pool overflowed before the merge
    (dead keys that another rank names) and a non-zero fourth colour channel; voxels of weight 0, 1 ... 2^20, tsdf +-1,
    -0, subnormals and rounding products in every case."""
    L = launches(mode, world)
    checks = []
    for name, root, color in MR.CASES:
        if name not in PLAIN:
            continue
        cid = MR.case_id(name, root, color)

        def one(cid=cid, name=name, root=root):
            recs, exp = _check_merge(L, cid, root)
            assert all(int(x["call0_rc"]) == 0 for x in recs), [int(x["call0_rc"]) for x in recs]
            pre_total = sum(len(x["pre_keys"]) for x in recs)
            if name == "all_empty":
                assert pre_total == 0
                assert all(str(x["call0_digest"]) == str(x["pre_digest"]) for x in recs), "an empty merge changed a volume"
            if name == "fill_exact":
                assert all(e.opened == len(e.lacking) and len(e.own) + e.opened == MR.SMALL_POOL for e in exp.values())
                assert all(int(recs[r]["call0_stats"][1]) == 0 for r in exp)
            if name in ("overflow", "pre_overflow"):
                assert all(int(recs[r]["call0_stats"][0]) == MR.SMALL_POOL for r in exp)
                assert any(e.drops[0] > 0 for e in exp.values())
            if name == "pre_overflow":
                assert len(_dead(recs[1])) > 0 and _dead(recs[1]) & set(_units(recs[0], "pre"))
            if name == "collide":
                assert any(k[0] in (-(1 << 20), (1 << 20) - 1) for x in recs for k in _units(x, "pre"))

        checks.append((cid, one))
    _run_all(checks)


@pytest.mark.parametrize("mode,world", MODES)
def test_workspace_protocol(launches, mode, world):
    """Scratch below the fixed part: GSB_ERR_WORKSPACE on every rank before any collective, no volume touched.  Scratch
    with the fixed part but not the payload: GSB_ERR_WORKSPACE on every rank with the same required size, the union's
    bricks opened and zero-filled on the receiving ranks; a retry with that size gives the bits a merge with ample scratch
    gives."""
    L = launches(mode, world)
    checks = []
    for root in MR.ROOTS:
        for color in (True, False):
            def below(root=root, color=color):
                cid = MR.case_id("ws_below_fixed", root, color)
                recs = [L.rec(cid, r) for r in range(world)]
                assert [int(x["call0_rc"]) for x in recs] == [GSB_ERR_WORKSPACE] * world
                req = {int(x["call0_required"]) for x in recs}
                assert len(req) == 1 and req.pop() > int(recs[0]["fixed"])
                assert all(str(x["call0_digest"]) == str(x["pre_digest"]) for x in recs)

            def fixed_then_retry(root=root, color=color):
                cid = MR.case_id("ws_fixed_then_retry", root, color)
                recs = [L.rec(cid, r) for r in range(world)]
                assert [int(x["call0_rc"]) for x in recs] == [GSB_ERR_WORKSPACE] * world
                dst = _dst(root, world)
                canon = 0 if dst is None else dst
                req = {int(x["call0_required"]) for x in recs}
                assert req == {int(recs[canon]["call0_need_own"])}, (req, int(recs[canon]["call0_need_own"]))
                # after the failed call: receiving ranks hold the union's bricks, the new ones zero-filled
                exp = merge_oracle([_units(x, "pre") for x in recs], dst, int(recs[0]["pool"]))
                for r in range(world):
                    if r in exp:
                        check_rank(exp[r], _units(recs[r], "call0"), int(recs[r]["call0_stats"][1] - recs[r]["pre_stats"][1]),
                                   set(), f"{cid} rank {r} after the failed call")
                        assert set(_units(recs[r], "call0")) == set().union(*(_units(x, "pre") for x in recs))
                    else:
                        assert str(recs[r]["call0_digest"]) == str(recs[r]["pre_digest"])
                # the retry
                assert [int(x["call1_rc"]) for x in recs] == [0] * world
                assert all(int(x["call1_bytes"]) == int(x["call0_required"]) for x in recs)
                _check_merge(L, cid, root, prefix="call1")
                ample = [L.rec(MR.case_id("partial", root, color), r) for r in range(world)]
                for r in range(world):
                    a, b = _units(recs[r], "call1"), _units(ample[r], "call0")
                    assert set(a) == set(b)
                    for k in a:
                        assert np.array_equal(a[k][0].view(np.uint32), b[k][0].view(np.uint32)), (r, k)
                        if color:
                            assert np.array_equal(a[k][1].view(np.uint32), b[k][1].view(np.uint32)), (r, k)

            checks += [(f"below_fixed-{root}-{color}", below), (f"fixed_then_retry-{root}-{color}", fixed_then_retry)]
    _run_all(checks)


@pytest.mark.parametrize("mode,world", MODES)
def test_reduce_across_ranks(launches, mode, world):
    """TSDFVolume.reduce_across_ranks: ranks whose pools differ in size agree on the largest before merging (the C call needs
    the same pool, colour setting and scratch size on every rank); volumes that disagree on colour raise ValueError on
    every rank and stay as they were; views integrated on every rank and merged equal the oracle of the ranks' exports."""
    L = launches(mode, world)
    checks = []
    pools = [MR.case_spec("unequal_pools", world, r)[0] for r in range(world)]
    for root in MR.ROOTS:
        for color in (True, False):
            def unequal(root=root, color=color):
                cid = MR.case_id("unequal_pools", root, color)
                recs, _ = _check_merge(L, cid, root, pool=max(pools))
                assert [int(x["pre_stats"][2]) for x in recs] == pools and len(set(pools)) > 1
                assert [int(x["call0_stats"][2]) for x in recs] == [max(pools)] * world
                assert all(str(x["error"]) == "" for x in recs)

            def end_to_end(root=root, color=color):
                cid = MR.case_id("end_to_end", root, color)
                recs, exp = _check_merge(L, cid, root)
                assert all(str(x["error"]) == "" for x in recs)
                assert min(len(x["pre_keys"]) for x in recs) > 20
                union = set().union(*(_units(x, "pre") for x in recs))
                assert len(union) > max(len(x["pre_keys"]) for x in recs)  # the shards overlap only in part
                for r in exp:
                    assert set(_units(recs[r], "call0")) == union

            checks += [(f"unequal-{root}-{color}", unequal), (f"end_to_end-{root}-{color}", end_to_end)]

    def mismatch():
        recs = [L.rec(MR.case_id("color_mismatch", "all", True), r) for r in range(world)]
        for x in recs:
            assert str(x["error"]).startswith("ValueError") and "with_color" in str(x["error"]), str(x["error"])
            assert str(x["call0_digest"]) == str(x["pre_digest"])

    checks.append(("color_mismatch", mismatch))
    _run_all(checks)
    print(f"{mode} {world} ranks: whole case list in {L.seconds:.1f} s")
