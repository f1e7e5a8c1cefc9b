"""Stream ordering of the WHENet forward: what each call waits for and what waits for it (whenet_api.cu forward_all,
whenet_set_stream, whenet_synchronize).

The kernels are checked elsewhere; here the same kernels run under the orchestration around them: caller streams, the legacy
default stream, switches between streams, one to four batch parts on internal streams, host inputs in one or several
passes with two calls in flight, and calls the library refuses.

Every result is compared bit for bit with per-crop references (angles and logits) from a fresh synchronous one-stream
context of the same precision and options, anchored once against float64.

Ordering is never detected by hoping a race corrupts data.  A hold (``torch.cuda._sleep``: a bounded spin of one thread)
delays everything queued after it on its stream, and every test that holds a stream asserts the hold is still running once
the dependent work has been queued, so a hold that ended early fails as inconclusive instead of passing unchecked.
- Data check: the hold sits on the caller's own stream before a producer (or consumer) of the forward's buffers, so the
  result is fixed: it equals the reference of what the producer wrote only if the forward waited for it.
- Event check: hold stream S1, queue call A there and record eA, queue call B on S2 and record eB; once eB has completed,
  eA must have completed too.
"""
import numpy as np
import pytest

from conftest import GOLD, SNAP
from elementwise_check import decode64
from test_gpu_batch_sweep import POOL, TOL, make_pool, mismatches, positions

pytestmark = pytest.mark.gpu

HOLD_CYCLES = 1 << 27                 # SM clock cycles: tens of milliseconds, far longer than queueing any call below
MAX_N = 512
# route: (precision, options) of the context under test and of its references
ROUTES = {"bf16": ("bf16", {}), "fp16": ("fp16", {}), "fp32": ("fp32", {}), "fp32_tc": ("fp32", {"tensor_cores": 1})}
H, W = 360, 640                       # frames of the crop scenarios
HELD_EARLY = "hold ended before the dependent work was queued"


# ----------------------------------------------------------------------------- helpers
def _torch():
    import torch
    return torch


def _model(route, max_batch=MAX_N, streams=1, **opts):
    import whenet_b200
    prec, ropts = ROUTES[route]
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=max_batch)
    m.set_option("streams", streams)
    for k, v in {**ropts, **opts}.items():
        m.set_option(k, v)
    return m


def _reference(route, crops):
    """Angles and logits of crops from a fresh synchronous one-stream context."""
    m = _model(route, 8, streams=1)
    try:
        return m._forward(np.ascontiguousarray(crops), want_logits=True)
    finally:
        m.close()


class Hold:
    """A bounded spin at the head of ``stream``: everything queued there after it waits for it."""

    def __init__(self, stream):
        torch = _torch()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(HOLD_CYCLES)
            self.ev = torch.cuda.Event()
            self.ev.record()

    def check(self):
        assert not self.ev.query(), HELD_EARLY


def _np(t):
    return t.cpu().numpy() if hasattr(t, "cpu") else np.asarray(t)


def _other(idx, k=17):
    """Other pool crops at every position."""
    return (np.asarray(idx) + k) % POOL


class Env:
    """The pool (host and device), its references per route, and buffers."""

    def __init__(self):
        torch = _torch()
        self.torch = torch
        self.pool = make_pool()
        self.dpool = torch.from_numpy(self.pool).cuda()
        self.refs = {r: _reference(r, self.pool) for r in ROUTES}
        torch.cuda._sleep(1)                   # the spin kernel is loaded before any hold is timed
        torch.cuda.synchronize()

    def device(self, idx):
        t = self.torch
        x = t.index_select(self.dpool, 0, t.from_numpy(np.asarray(idx, np.int64)).cuda())
        t.cuda.synchronize()                   # written on torch's stream, read on the context's
        return x

    def pinned(self, idx):
        return self.torch.from_numpy(np.ascontiguousarray(self.pool[np.asarray(idx)])).pin_memory()

    def outs(self, n, pinned=False):
        """NaN-filled angle and logit buffers, on the device or pinned on the host."""
        t = self.torch
        kw = dict(pin_memory=True) if pinned else dict(device="cuda")
        y = t.full((n, 3), float("nan"), dtype=t.float32, **kw)
        lg = t.full((n, 252), float("nan"), dtype=t.float32, **kw)
        t.cuda.synchronize()
        return y, lg

    def bad(self, route, idx, y, lg):
        """Positions whose angles or logits differ in any bit from their pool crop's reference."""
        ref_ang, ref_lg = self.refs[route]
        return mismatches(ref_ang, ref_lg, np.asarray(idx), _np(y), _np(lg)).tolist()


@pytest.fixture(scope="module")
def env():
    e = Env()
    yield e
    e.torch.cuda.synchronize()


def _frames(seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (2, H, W, 3), dtype=np.uint8)


RECTS = np.array([[0, H, 0, W], [10, 200, 30, 330], [100, 101, 200, 201], [5, 229, 7, 231], [300, 360, 600, 640],
                  [0, 2, 0, 3], [50, 300, 400, 500], [120, 359, 1, 639]], np.int32)
BOXES = np.array([[20.5, 30.2, 180.7, 200.9], [0, 0, H, W], [100.1, 300.4, 250.8, 420.3], [300.5, 500.5, 359.9, 639.9],
                  [5, 5, 60, 40], [200, 100, 340, 260], [40.7, 560.1, 150.2, 630.6], [150, 250, 210, 330]], np.float32)


def _cv2_crops(frame, rects):
    cv2 = pytest.importorskip("cv2")
    return np.stack([cv2.resize(cv2.cvtColor(frame[y0:y1, x0:x1], cv2.COLOR_BGR2RGB), (224, 224)) for y0, y1, x0, x1 in rects])


def _box_rects(boxes):
    from whenet_b200 import crops
    return np.array([crops.enlarge_box(b, H, W) for b in boxes], np.int32)


def _crop_resize(m, frame, out):
    from whenet_b200._lib import check
    from whenet_b200.whenet import _ptr
    check(m._L.whenet_crop_resize_u8(m._h, _ptr(frame), H, W, 1, _ptr(RECTS), len(RECTS), 1, _ptr(out)))


def _crop_boxes(m, frame, out, rects_out, valid_out):
    from whenet_b200._lib import check
    from whenet_b200.whenet import _ptr
    frame_of = np.zeros(len(BOXES), np.int32)
    check(m._L.whenet_crop_boxes_u8(m._h, _ptr(frame), 1, H, W, 1, _ptr(BOXES), _ptr(frame_of), len(BOXES), 1, _ptr(out),
                                    _ptr(rects_out), _ptr(valid_out)))


# ----------------------------------------------------------------------------- references
@pytest.mark.parametrize("route", list(ROUTES))
def test_references_anchor(env, route):
    """The references of the Sample crops against the committed float64 logits: logits within the suite's fp32 bound
    (2e-3), angles within the route's parity tolerance; every pool reference finite."""
    ang, lg = env.refs[route]
    assert np.isfinite(ang).all() and np.isfinite(lg).all()
    gold = np.load(GOLD + "/sample_logits_f64.npy")
    assert np.array_equal(env.pool[:2], np.load(GOLD + "/sample_crops.npy"))
    ref_ang = np.stack(decode64([gold[:, :120], gold[:, 120:186], gold[:, 186:]]), axis=1)
    d = np.abs(ang[:2].astype(np.float64) - ref_ang)
    d = np.minimum(d, 360 - d).max()
    prec = ROUTES[route][0]
    assert d <= TOL[prec], (route, d)
    if prec == "fp32":
        assert np.abs(lg[:2].astype(np.float64) - gold).max() < 2e-3, route


# ----------------------------------------------------------------------------- (a) producer on the caller stream
def _producer_device(env, m, route, S, n, streams, what):
    """On S: hold, overwrite x (crops A) with crops B; forward_device on S must give ref(B)."""
    torch = env.torch
    m.set_option("streams", streams)
    ia = positions(n)
    ib = _other(ia)
    x, xb = env.device(ia), env.device(ib)
    y, lg = env.outs(n)
    m.forward_device(x, y, lg)                 # warm-up (also captures the graph when graph replay is on)
    torch.cuda.synchronize()
    bad = []
    if env.bad(route, ia, y, lg):
        bad.append((what, streams, n, "warm-up"))
    h = Hold(S)
    with torch.cuda.stream(S):
        x.copy_(xb)
    m.forward_device(x, y, lg)
    h.check()
    torch.cuda.synchronize()
    p = env.bad(route, ib, y, lg)
    if p:
        bad.append((what, streams, n, "positions %s" % p[:4]))
    return bad


@pytest.mark.parametrize("route", list(ROUTES))
def test_producer_on_caller_stream(env, route):
    """Crops written on the caller's stream behind a hold are what forward_device reads: streams 1-4 at n = 8, 64, 131 and
    512 (two to four parts from 64 crops), a replayed graph, the legacy default stream; forward_host_to_device writes its
    device outputs only after the caller's earlier work on the stream (NaN fills behind a hold)."""
    torch = env.torch
    S = torch.cuda.Stream()
    m = _model(route)
    bad = []
    try:
        m.set_stream(S.cuda_stream)
        for streams in (1, 2, 3, 4):
            for n in (8, 64, 131, 512):
                bad += _producer_device(env, m, route, S, n, streams, "device")
        m.set_option("graph", 1)
        for n in (8, 131):
            bad += _producer_device(env, m, route, S, n, 2, "graph")
        m.set_option("graph", 0)
        m.set_stream(0)                        # torch's default stream: cudaStreamLegacy
        for n in (8, 131):
            bad += _producer_device(env, m, route, torch.cuda.default_stream(), n, 2, "legacy stream")
        m.set_stream(S.cuda_stream)
        for streams in (1, 2, 3, 4):
            for n in (8, 131, 512):
                m.set_option("streams", streams)
                ia = positions(n)
                ib = _other(ia)
                xh = env.pinned(ia)
                y, lg = env.outs(n)
                m.forward_host_to_device(xh, y, lg)
                m.synchronize()
                if env.bad(route, ia, y, lg):
                    bad.append(("host_to_device", streams, n, "warm-up"))
                xh.numpy()[:] = env.pool[ib]           # host write: the previous upload has completed
                h = Hold(S)
                with torch.cuda.stream(S):
                    y.fill_(float("nan"))
                    lg.fill_(float("nan"))
                m.forward_host_to_device(xh, y, lg)
                h.check()
                torch.cuda.synchronize()
                p = env.bad(route, ib, y, lg)
                if p:
                    bad.append(("host_to_device", streams, n, "positions %s" % p[:4]))
    finally:
        torch.cuda.synchronize()
        m.close()
    assert not bad, (route, bad[:8])


@pytest.mark.parametrize("entry", ["crop_resize", "crop_boxes"])
def test_producer_of_frames_on_caller_stream(env, entry):
    """A device frame overwritten on the caller's stream behind a hold, then cropped (whenet_crop_resize_u8 or
    whenet_crop_boxes_u8) and the crops run through forward_device on that stream: the crops are cv2's crops of the new
    frame and the results the references of those crops."""
    torch = env.torch
    fa, fb = _frames(11 if entry == "crop_resize" else 12)
    rects = RECTS if entry == "crop_resize" else _box_rects(BOXES)
    refs = {}
    for key, f in (("a", fa), ("b", fb)):
        c = _cv2_crops(f, rects)
        refs[key] = (c,) + tuple(_reference("bf16", c))
    k = len(rects)
    S = torch.cuda.Stream()
    m = _model("bf16", 64, streams=2)
    try:
        m.set_stream(S.cuda_stream)
        frame, frame_b = torch.from_numpy(fa).cuda(), torch.from_numpy(fb).cuda()
        crops = torch.empty((k, 224, 224, 3), dtype=torch.uint8, device="cuda")
        y, lg = env.outs(k)
        rects_out = np.full((k, 4), -1, np.int32)
        valid_out = np.full(k, -1, np.int32)

        def call():
            if entry == "crop_resize":
                _crop_resize(m, frame, crops)
            else:
                _crop_boxes(m, frame, crops, rects_out, valid_out)
            m.forward_device(crops, y, lg)

        for key in ("a", "b"):
            if key == "a":
                call()                                 # warm-up on frame A
            else:
                h = Hold(S)
                with torch.cuda.stream(S):
                    frame.copy_(frame_b)
                call()
                h.check()
            torch.cuda.synchronize()
            c, ang, lgr = refs[key]
            assert np.array_equal(crops.cpu().numpy(), c), (entry, key)
            assert np.array_equal(y.cpu().numpy().view(np.uint32), ang.view(np.uint32)), (entry, key)
            assert np.array_equal(lg.cpu().numpy().view(np.uint32), lgr.view(np.uint32)), (entry, key)
            if entry == "crop_boxes":
                assert np.array_equal(rects_out, rects) and valid_out.tolist() == [1] * k
    finally:
        torch.cuda.synchronize()
        m.close()


# ----------------------------------------------------------------------------- (b) consumer on the caller stream
@pytest.mark.parametrize("route", list(ROUTES))
def test_consumer_on_caller_stream(env, route):
    """The join of a two- to four-part pass: on the caller's stream, behind a hold, the outputs are filled with NaN, the
    forward is queued and the outputs are copied right after it; the copies equal the references.  Device and pinned-host
    inputs at n = 64, 65, 131, 256 and 512."""
    torch = env.torch
    S = torch.cuda.Stream()
    m = _model(route)
    bad = []
    try:
        m.set_stream(S.cuda_stream)
        for streams in (2, 3, 4):
            m.set_option("streams", streams)
            for n in (64, 65, 131, 256, 512):
                idx = positions(n)
                for kind in ("device", "pinned"):
                    x = env.device(idx) if kind == "device" else env.pinned(idx)
                    fwd = m.forward_device if kind == "device" else m.forward_host_to_device
                    y, lg = env.outs(n)
                    fwd(x, y, lg)                      # warm-up
                    torch.cuda.synchronize()
                    h = Hold(S)
                    with torch.cuda.stream(S):
                        y.fill_(float("nan"))
                        lg.fill_(float("nan"))
                        fwd(x, y, lg)
                        snap, snap_l = y.clone(), lg.clone()
                    h.check()
                    torch.cuda.synchronize()
                    p = env.bad(route, idx, snap, snap_l)
                    if p:
                        bad.append((kind, streams, n, "positions %s" % p[:4]))
    finally:
        torch.cuda.synchronize()
        m.close()
    assert not bad, (route, bad[:8])


# ----------------------------------------------------------------------------- (c) stream switch
class Call:
    """One call of a kind on its own inputs and outputs, with the references of its results."""

    def __init__(self, env, m, kind, seed):
        torch = env.torch
        self.env, self.m, self.kind = env, m, kind
        self.n = 131 if kind == "device131" else 8
        self.idx = np.random.default_rng(seed).permutation(POOL)[:self.n] if self.n <= POOL else \
            np.random.default_rng(seed).integers(0, POOL, self.n)
        self.ref = None
        if kind == "host_async":
            self.x = env.pinned(self.idx)
            self.y, self.lg = env.outs(self.n, pinned=True)
        elif kind == "crops":
            f = _frames(seed)[0]
            c = _cv2_crops(f, RECTS)
            self.crops_ref = c
            self.ref = tuple(_reference("bf16", c))
            self.frame = torch.from_numpy(f).cuda()
            self.x = torch.empty((len(RECTS), 224, 224, 3), dtype=torch.uint8, device="cuda")
            self.y, self.lg = env.outs(len(RECTS))
        else:
            self.x = env.device(self.idx)
            self.y, self.lg = env.outs(self.n)

    def __call__(self):
        if self.kind == "host_async":
            self.m.forward_host_async(self.x, self.y, self.lg)
        elif self.kind == "crops":
            _crop_resize(self.m, self.frame, self.x)
            self.m.forward_device(self.x, self.y, self.lg)
        else:
            self.m.forward_device(self.x, self.y, self.lg)

    def clear(self):
        self.y.fill_(float("nan"))
        self.lg.fill_(float("nan"))
        self.env.torch.cuda.synchronize()

    def bad(self):
        if self.kind == "crops":
            ok = np.array_equal(self.x.cpu().numpy(), self.crops_ref) and \
                np.array_equal(_np(self.y).view(np.uint32), self.ref[0].view(np.uint32)) and \
                np.array_equal(_np(self.lg).view(np.uint32), self.ref[1].view(np.uint32))
            return [] if ok else ["crops or results"]
        return self.env.bad("bf16", self.idx, self.y, self.lg)


# (call A, call B).  Two two-part calls also queue their parts one after the other on the same internal streams; a
# two-part call followed by a one-pass call shares only the workspace.
SWITCH_PAIRS = [("device8", "device8"), ("device131", "device131"), ("device131", "device8"), ("graph", "graph"),
                ("host_async", "host_async"), ("crops", "crops")]


@pytest.mark.parametrize("kind_a,kind_b", SWITCH_PAIRS)
def test_stream_switch_orders_work(env, kind_a, kind_b):
    """Call A queued on S1 behind a hold, set_stream(S2), call B on S2: once B's event has completed, A's has too, and
    both results equal their references.  forward_device at n = 8 and at n = 131 on two streams, graph replays captured on
    S1 and replayed on S2, forward_host_async with pinned buffers, crop_resize followed by a forward."""
    torch = env.torch
    S1, S2 = torch.cuda.Stream(), torch.cuda.Stream()
    m = _model("bf16", 256, streams=2, graph=int(kind_a == "graph"))
    try:
        a, b = Call(env, m, kind_a, 1), Call(env, m, kind_b, 2)
        m.set_stream(S1.cuda_stream)
        a()
        b()                                    # warm-up on S1 (graph replay: both graphs are captured on S1)
        m.synchronize()
        torch.cuda.synchronize()
        assert not a.bad() and not b.bad(), "warm-up"
        a.clear()
        b.clear()
        h = Hold(S1)
        a()
        ea = torch.cuda.Event()
        ea.record(S1)
        m.set_stream(S2.cuda_stream)
        b()
        eb = torch.cuda.Event()
        eb.record(S2)
        h.check()
        eb.synchronize()
        a_done = ea.query()
        torch.cuda.synchronize()
        assert a_done, "call B on S2 completed while call A on S1 had not: set_stream did not order S2 after S1"
        assert not a.bad() and not b.bad(), (a.bad()[:4], b.bad()[:4])
    finally:
        torch.cuda.synchronize()
        m.close()


def test_switch_back_to_internal_stream(env):
    """Call A on S1 behind a hold, set_stream(None), call B on the internal stream: synchronize() returns only after A has
    completed, and both results equal their references."""
    torch = env.torch
    S1 = torch.cuda.Stream()
    m = _model("bf16", 256, streams=2)
    try:
        a, b = Call(env, m, "device131", 3), Call(env, m, "device8", 4)
        m.set_stream(S1.cuda_stream)
        a()
        b()
        m.synchronize()
        a.clear()
        b.clear()
        h = Hold(S1)
        a()
        ea = torch.cuda.Event()
        ea.record(S1)
        m.set_stream(None)
        b()
        h.check()
        m.synchronize()
        a_done = ea.query()
        torch.cuda.synchronize()
        assert a_done, "synchronize() on the internal stream returned while call A on S1 had not completed"
        assert not a.bad() and not b.bad(), (a.bad()[:4], b.bad()[:4])
    finally:
        torch.cuda.synchronize()
        m.close()


def test_synchronize_after_switch_covers_old_stream(env):
    """forward_host_async queued on S1 behind a hold, set_stream(S2), synchronize(): the host outputs are written."""
    torch = env.torch
    S1, S2 = torch.cuda.Stream(), torch.cuda.Stream()
    m = _model("bf16", 256, streams=2)
    try:
        a = Call(env, m, "host_async", 5)
        m.set_stream(S1.cuda_stream)
        a()
        m.synchronize()
        a.clear()
        h = Hold(S1)
        a()
        m.set_stream(S2.cuda_stream)
        h.check()
        m.synchronize()
        got = a.bad()
        nan = int(np.isnan(_np(a.y)).any(axis=1).sum())
        torch.cuda.synchronize()
        assert not got, "after set_stream(S2) and synchronize(): %d of %d crops still NaN, %d differ" % (nan, a.n, len(got))
    finally:
        torch.cuda.synchronize()
        m.close()


# ----------------------------------------------------------------------------- (d) batch parts
PART_NS = (63, 64, 65, 96, 127, 128, 131, 136, 192, 255, 256, 257, 511, 512)


@pytest.mark.parametrize("route", list(ROUTES))
def test_batch_parts_bitwise(env, route):
    """streams 1-4 (one to four batch parts, each on its own route by its own size) at n around the part and route
    switches: device, pinned-host and pageable-host inputs (threaded staging from 56 crops per part), every crop equal to
    its reference.  The launch count grows with the part count from 64 crops and stays put below."""
    torch = env.torch
    m = _model(route)
    bad, launches = [], {}
    xh = torch.empty((MAX_N, 224, 224, 3), dtype=torch.uint8, pin_memory=True)
    ah, lh = env.outs(MAX_N, pinned=True)
    try:
        for streams in (1, 2, 3, 4):
            m.set_option("streams", streams)
            for n in PART_NS:
                idx = positions(n)
                x = env.device(idx)
                y, lg = env.outs(n)
                l0 = m.launch_count()
                m.forward_device(x, y, lg)
                m.synchronize()
                launches[streams, n] = m.launch_count() - l0
                p = env.bad(route, idx, y, lg)
                if p:
                    bad.append(("device", streams, n, p[:4]))
                xh[:n].numpy()[:] = env.pool[idx]
                ah.fill_(float("nan"))
                lh.fill_(float("nan"))
                m.forward_host(xh[:n], ah[:n], lh[:n])
                p = env.bad(route, idx, ah[:n], lh[:n])
                if p:
                    bad.append(("pinned", streams, n, p[:4]))
                if n >= 56:
                    ang, lgp = m._forward(np.ascontiguousarray(env.pool[idx]), want_logits=True)
                    p = env.bad(route, idx, ang, lgp)
                    if p:
                        bad.append(("pageable", streams, n, p[:4]))
    finally:
        torch.cuda.synchronize()
        m.close()
    assert not bad, (route, bad[:8])
    for n in PART_NS:
        counts = [launches[s, n] for s in (1, 2, 3, 4)]
        if n >= 64:
            assert all(u < v for u, v in zip(counts, counts[1:])), (route, n, counts)
        else:
            assert len(set(counts)) == 1, (route, n, counts)


# ----------------------------------------------------------------------------- (e) in-flight host calls
@pytest.mark.parametrize("host_chunk", [None, 1, 7, 64])
def test_async_host_pairs(env, host_chunk):
    """Two forward_host_async calls in flight (the header's limit) at n = 1, 8, 63, 64, 131 and 512 on 1-4 streams, whole
    passes or passes of host_chunk crops (odd and even pass counts flip the staging slot parity); then both pinned inputs
    are overwritten with other crops and queued again: the results follow the new contents."""
    torch = env.torch
    m = _model("bf16", streams=1, **({} if host_chunk is None else {"host_chunk": host_chunk}))
    bad = []
    bufs = [torch.empty((MAX_N, 224, 224, 3), dtype=torch.uint8, pin_memory=True) for _ in range(2)]
    outs = [env.outs(MAX_N, pinned=True) for _ in range(2)]
    try:
        for streams in (1, 2, 3, 4):
            m.set_option("streams", streams)
            for n in (1, 8, 63, 64, 131, 512):
                ia = positions(n)
                sets = [(ia, _other(ia, 5)), (_other(ia, 11), _other(ia, 23))]
                for rnd, pair in enumerate(sets):
                    for buf, (y, lg), idx in zip(bufs, outs, pair):
                        buf[:n].numpy()[:] = env.pool[idx]       # after a synchronize: no call reads the buffers
                        y.fill_(float("nan"))
                        lg.fill_(float("nan"))
                    for buf, (y, lg) in zip(bufs, outs):
                        m.forward_host_async(buf[:n], y[:n], lg[:n])
                    m.synchronize()
                    for k, ((y, lg), idx) in enumerate(zip(outs, pair)):
                        p = env.bad("bf16", idx, y[:n], lg[:n])
                        if p:
                            bad.append((streams, n, "round %d call %d" % (rnd, k), p[:4]))
    finally:
        torch.cuda.synchronize()
        m.close()
    assert not bad, (host_chunk, bad[:8])


@pytest.mark.parametrize("streams,n,host_chunk", [(3, 131, None), (1, 63, 7)])
def test_async_host_ten_pairs(env, streams, n, host_chunk):
    """Ten pairs of forward_host_async calls, each pair on new crops into its own output buffers: every output equals its
    crops' references."""
    torch = env.torch
    m = _model("bf16", 256, streams=streams, **({} if host_chunk is None else {"host_chunk": host_chunk}))
    rng = np.random.default_rng(77)
    bufs = [torch.empty((n, 224, 224, 3), dtype=torch.uint8, pin_memory=True) for _ in range(2)]
    outs = [env.outs(n, pinned=True) for _ in range(20)]
    idxs = [rng.integers(0, POOL, n) for _ in range(20)]
    try:
        for k in range(10):
            for j in (0, 1):
                bufs[j].numpy()[:] = env.pool[idxs[2 * k + j]]
            for j in (0, 1):
                m.forward_host_async(bufs[j], *outs[2 * k + j])
            m.synchronize()
    finally:
        torch.cuda.synchronize()
        m.close()
    bad = [(k, p[:4]) for k, ((y, lg), idx) in enumerate(zip(outs, idxs)) if (p := env.bad("bf16", idx, y, lg))]
    assert not bad, bad


# ----------------------------------------------------------------------------- (f) refused calls
def test_refused_calls_keep_stream(env):
    """Calls refused with WHENET_EINVAL after set_stream(S) (n > max_batch; a tapped crop outside the call) leave the
    context on S: crops written on S behind a hold are still what the next forwards read, and a four-part forward at
    n = 512 equals its references."""
    from whenet_b200 import WhenetError
    from whenet_b200.whenet import _ptr
    torch = env.torch
    S = torch.cuda.Stream()
    m = _model("bf16", streams=4)
    try:
        m.set_stream(S.cuda_stream)
        x = torch.zeros((MAX_N + 1, 224, 224, 3), dtype=torch.uint8, device="cuda")      # large enough for n + 1
        y = torch.zeros((MAX_N + 1, 3), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        rc = m._L.whenet_forward_u8(m._h, _ptr(x), MAX_N + 1, 1, _ptr(y), None, 1)
        assert rc == -1 and b"max_batch" in m._L.whenet_last_error()
        m.enable_taps(True, faithful=True, crops=[100])
        with pytest.raises(WhenetError) as e:
            m.forward_device(x[:8], y[:8])
        assert e.value.code == -1 and "outside" in str(e.value)
        m.enable_taps(False)
        bad = []
        for n in (8, 131, 512):
            bad += _producer_device(env, m, "bf16", S, n, 4, "after refused calls")
    finally:
        torch.cuda.synchronize()
        m.close()
    assert not bad, bad
