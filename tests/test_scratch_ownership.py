"""CPU test of who owns the rasterizer's scratch blocks and on which streams they are used (gs2mesh_b200/rasterizer.py
`Scratch`, gs2mesh_b200/renderer.py stream sets).

The REAL `render_image_pair`, `_enqueue_pair`, `rasterize_forward_pair` and `rasterize_forward` run against the fake CUDA
streams and events of tests/test_stream_schedule.py, on CPU tensors.  The library is replaced by a stub that enqueues the
workspace accesses `gsb_raster_forward_pair` makes (csrc/gsb_raster.cu): the fused preprocess writes both eyes' blocks on
the left stream; the right eye continues on its own stream behind an event and, with a shared depth order, reads the left
eye's depth order from the left block."""
import contextlib

import pytest
import torch

from gs2mesh_b200 import _lib
from gs2mesh_b200 import rasterizer as rast
from gs2mesh_b200 import renderer as rmod
from tests import test_stream_schedule as tss
from tests.test_stream_schedule import fake_cuda  # noqa: F401  (fixture)

P, W, H, N_VIEWS = 8, 64, 48, 4


class FakeLib:
    """The library entry points the wrappers call.  `uses` collects (workspace address, stream handle) for every stream a
    workspace is enqueued on."""

    def __init__(self, streams):
        self.streams = streams  # handle -> fake stream
        self.uses = []
        self.crossed = []  # (workspace, stream handle) of a block used on the other eye's stream
        self.views = []  # workspace of every single-view call

    def gsb_raster_workspace_bytes(self, P, W, H, cap):
        return 256 + cap

    def gsb_raster_forward(self, args, stream):
        a = args._obj
        self.streams[stream.value].op("frame", access=[((a.workspace, "shared"), True), ((a.workspace, "eye"), True)])
        self.uses.append((a.workspace, stream.value))
        self.views.append(a.workspace)
        return _lib.GSB_OK

    def gsb_raster_forward_pair(self, left, right, stream_left, stream_right):
        wl, wr = left._obj.workspace, right._obj.workspace
        shared = bool(left._obj.flags & _lib.RASTER_PAIR_SHARED_DEPTH)
        sl, sr = self.streams[stream_left.value], self.streams[stream_right.value]
        # each block as its shared part (preprocess results, depth order) and the part its eye's binning writes
        sl.op("pair: preprocess (+ depth sort)", access=[((wl, "shared"), True), ((wr, "shared"), True)])
        if sr is not sl:
            sr.wait_event(sl.record_event())
        sl.op("bin + blend L", access=[((wl, "shared"), False), ((wl, "eye"), True)])
        sr.op("bin + blend R", access=[((wr, "shared"), False), ((wr, "eye"), True)] + ([((wl, "shared"), False)] if shared else []))
        self.crossed += [(wr, sl.cuda_stream)] + ([(wl, sr.cuda_stream)] if shared else [])
        self.uses += [(wl, sl.cuda_stream), (wr, sr.cuda_stream)] + self.crossed[-1 - shared:]
        return _lib.GSB_OK


@pytest.fixture
def fake_lib(fake_cuda, monkeypatch):
    streams = {fake_cuda.cuda_stream: fake_cuda}

    class Stream(tss.FakeStream):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            streams[self.cuda_stream] = self

    recorded, kept = set(), []

    def record_stream(t, s):
        kept.append(t)  # keeps every workspace address unique for the race check
        recorded.add((t.data_ptr(), s.cuda_stream))

    lib = FakeLib(streams)
    lib.recorded = recorded
    monkeypatch.setattr(torch.cuda, "Stream", Stream)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.Tensor, "record_stream", record_stream)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda t: True))
    monkeypatch.setattr(_lib, "lib", lambda: lib)
    monkeypatch.setattr(rast, "image_to_u8", lambda chw, out=None: out)
    return lib


class _View:
    width, height, tan_fovx, tan_fovy = W, H, 0.5, 0.4


def make_renderer(in_flight=2, overlap_eyes=True):
    r = rmod.Renderer.from_scene([dict(left={}, right={}) for _ in range(N_VIEWS)], 0.1, None)
    r.pairs_in_flight, r.spare_buffer_sets, r.copy_streams, r.overlap_eyes = in_flight, 0, False, overlap_eyes
    r._views = [[_View(), _View()] for _ in range(N_VIEWS)]
    r._camera_table = torch.zeros(N_VIEWS, 2, 36)
    r.means3D, r.opacity, r.shs = torch.zeros(P, 3), torch.zeros(P), torch.zeros(P, 16, 3)
    r.scales, r.rotations, r.sh_degree, r.background = torch.zeros(P, 3), torch.zeros(P, 4), 3, torch.zeros(3)
    r._status = torch.zeros(N_VIEWS, 2, 4, dtype=torch.int64)
    r._shared_depth = [True, False] * (N_VIEWS // 2)
    r._min_instances = 0
    r._view_block = rast.Scratch("cpu")
    r._serial_blocks = (r._view_block, rast.Scratch("cpu"))
    r._ready = True
    bufs = {}

    def buffers(w, h, parity=0):
        if parity not in bufs:
            img = lambda: [torch.zeros(3, h, w), torch.zeros(3, h, w)]
            bufs[parity] = dict(color=img(), u8=img(), depth=torch.zeros(h, w), final_T=torch.zeros(h, w), host_u8=img())
        return bufs[parity]

    r._buffers = buffers
    return r


def lagged_loop(r, calls=10):
    """bench.py's host-buffer loop: pair n is waited for after pair n + pairs_in_flight was enqueued."""
    views = [n % N_VIEWS for n in range(calls)]
    lag = max(1, r.pairs_in_flight)
    pending = [r.render_image_pair(v, to_host=True, wait=False) for v in views[:lag]]
    for n in range(calls):
        out = pending.pop(0)
        if n + lag < calls:
            pending.append(r.render_image_pair(views[n + lag], to_host=True, wait=False))
        out["ready"].synchronize()


@pytest.mark.parametrize("overlap_eyes", [True, False])
@pytest.mark.parametrize("mode", ["fused", "noshare", "separate"])
def test_blocks_are_recorded_on_every_stream_they_are_enqueued_on(fake_lib, monkeypatch, mode, overlap_eyes):
    """Every (block, stream) the library is handed -- including the right eye's block on the left stream, and under a
    shared depth order the left eye's block on the right stream -- is recorded; and no two frames touch one block
    unordered, also when the next pair of a stream set is enqueued before the previous one was waited for."""
    monkeypatch.setenv("GSB_PAIR_MODE", mode)
    r = make_renderer(overlap_eyes=overlap_eyes)
    lagged_loop(r)
    assert fake_lib.uses and set(fake_lib.uses) <= fake_lib.recorded
    if mode != "separate" and overlap_eyes:
        assert len(fake_lib.crossed) == 10 + 5 * (mode == "fused")  # every pair; the shared depth order of every other
    assert tss.G.races() == []


def test_separate_mode_renders_the_eyes_in_the_sets_blocks(fake_lib, monkeypatch):
    """`separate` renders both eyes through render_view at the same time, on the two streams of a set: each eye gets its
    set's own block, never the renderer's single-view block."""
    monkeypatch.setenv("GSB_PAIR_MODE", "separate")
    r = make_renderer()
    lagged_loop(r, calls=4)
    views = fake_lib.views
    assert len(views) == 8
    sets = [tuple(s.scratch[e].workspace.data_ptr() for e in range(2)) for s in r._stream_sets]
    assert len({ws for pair in sets for ws in pair}) == 4  # two sets, two eyes: four blocks
    for n in range(4):
        assert (views[2 * n], views[2 * n + 1]) == sets[n % 2]
    assert r._view_block.workspace is None


def test_growing_one_sets_blocks_leaves_the_other_sets_alone(fake_lib):
    r = make_renderer(in_flight=2)
    r.render_image_pair(0, to_host=True, wait=False)
    r.render_image_pair(1, to_host=True, wait=False)
    a, b = r._stream_sets
    before = {id(s): (s.workspace, s.max_instances) for s in a.scratch + b.scratch}
    r._min_instances = 10 * max(s.max_instances for s in a.scratch)
    r.render_image_pair(2, to_host=True, wait=False)  # set a again, with a larger capacity
    for s in a.scratch:
        assert s.max_instances == r._min_instances and s.workspace is not before[id(s)][0]
    for s in b.scratch:
        assert (s.workspace, s.max_instances) == before[id(s)]
    assert set(fake_lib.uses) <= fake_lib.recorded


def test_asynchronous_calls_need_their_own_blocks(fake_lib):
    view = dict(means3D=torch.zeros(P, 3), opacities=torch.zeros(P), viewmatrix=torch.eye(4), projmatrix=torch.eye(4),
                campos=torch.zeros(3), bg=torch.zeros(3), width=W, height=H, tan_fovx=0.5, tan_fovy=0.4,
                shs=torch.zeros(P, 16, 3), scales=torch.zeros(P, 3), rotations=torch.zeros(P, 4), sh_degree=3)
    with pytest.raises(ValueError):
        rast.rasterize_forward(**view, async_mode=True)
    with pytest.raises(ValueError):  # the bit decides, not the keyword
        rast.rasterize_forward(**view, flags=rast.DEFAULT_FLAGS | _lib.RASTER_ASYNC)
    eye = dict(viewmatrix=torch.eye(4), projmatrix=torch.eye(4), campos=torch.zeros(3), tan_fovx=0.5, tan_fovy=0.4,
               out_color=torch.zeros(3, H, W))
    st = torch.cuda.current_stream()
    with pytest.raises(ValueError):
        rast.rasterize_forward_pair(means3D=view["means3D"], opacities=view["opacities"], shs=view["shs"], scales=view["scales"],
                                    rotations=view["rotations"], sh_degree=3, bg=view["bg"], width=W, height=H,
                                    eyes=[eye, dict(eye)], streams=(st, st))
    assert fake_lib.uses == []
