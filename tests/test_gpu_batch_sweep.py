"""The WHENet forward at every batch size: the same bits for every crop across each batch-size route switch (DESIGN §4.2).

The forward picks kernels from the crops per pass (two half-batch streams from 64 crops, batched SE and head kernels from 64
crops per pass, the KD expand on chip or as a GEMM, K1X or split K1, K2 or pw_tc2, the SE tail).  Each crop's angles and
logits must not depend on which of them ran, nor on its position in the batch.

- A pool of 48 distinct crops gets per-crop references from a fresh 8-crop context, checked against the float64 oracle.
- At every swept n a seeded permutation of the pool runs through forward_device; every position must equal its crop's
  reference bit for bit, angles and logits.
- ``routes`` restates the launcher's batch-size rules.  Its launch count and profile layer names are asserted at every
  swept n, and it generates the switch points that the sweep must cross from both sides.
- At the route switches, faithful taps on edge crops must equal the same crop's 8-crop taps.
- Host inputs (pageable and pinned), Python chunking, ragged passes, the graph cache and the tensor-map caches past their
  limits give the same bits.
- Negative controls show that the comparison reports a one-ulp change and a legitimately different rounding.
"""
import os
import re
import subprocess
import time

import numpy as np
import pytest

import elementwise_check as ec
import whenet_bounds as wb
from conftest import GOLD, ROOT, SNAP
from whenet_b200 import arch

gpu = pytest.mark.gpu

BLOCKS = {b.idx: b for b in arch.blocks()}
SPLIT_CTAS = 120                       # option k1_split_ctas: split a crop's chunks over CTAs until the grid has this many
# K1 tile plans (kernels_fused.cuh plan_k1; pinned by test_route_model_plans): output tiles per crop, crops per CTA, chunks
K1_PLAN = {2: (49, 1, 2), 3: (16, 1, 3), 4: (16, 1, 3), 5: (4, 1, 5), 6: (4, 1, 3), 7: (1, 1, 5), 8: (1, 1, 5), 9: (1, 1, 5),
           10: (1, 1, 6), 11: (1, 1, 6), 12: (1, 1, 6), 13: (1, 2, 18), 14: (1, 2, 18), 15: (1, 2, 18), 16: (1, 2, 12)}
K1X_BLOCKS = (2, 3, 4, 6)
KD_CHUNKS = {7: 15, 8: 15, 9: 15, 10: 21, 11: 21, 12: 7, 13: 9, 14: 9, 15: 9, 16: 9}    # bf16 KD, blocks 7-16 (dwse_chunk)
B1_KD_TILES = 64                       # bf16 block 1 on KD: 14x14 spatial tiles of the 112x112 map
MAX_N = 512
POOL = 48
TOL = {"bf16": 0.6, "fp16": 0.08, "fp32": 0.01}      # DESIGN §2, degrees
TAP_POOL = [0, 8, 10, 40]              # pool crops whose taps are compared: Sample, all 0, checkerboard, uniform random
SYNTHETIC = list(range(8, 15))         # all 0, all 255, checkerboard, four gradients

# route: (precision, options, streams)
ROUTES = {
    "bf16": ("bf16", {}, 2),
    "bf16_1stream": ("bf16", {}, 1),
    "fp16": ("fp16", {}, 2),
    "fp32_split": ("fp32", {"tensor_cores": 1}, 2),
    "fp32_cuda": ("fp32", {"tensor_cores": 0}, 2),
}


# ----------------------------------------------------------------------------- route model (whenet_api.cu forward_all / run_dw_route / launch_pw)
def _cdiv(a, b):
    return -(-a // b)


def _col_tile(n_cols, cap):
    """Column tile of a 1x1 conv with at most ``cap`` columns per tile (plan_k2, launch_pw_tc2)."""
    nt = n_cols
    parts = _cdiv(n_cols, cap)
    while nt > cap:
        nt = (_cdiv(n_cols, parts) + 15) & ~15
        parts += 1
    return (nt + 15) & ~15


def k2_tiles(m_rows, n_cols):
    """plan_k2's tile count: 128-row tiles times <= 64-column tiles."""
    return _cdiv(m_rows, 128) * _cdiv(n_cols, _col_tile(n_cols, 64))


def pw_tc2_tile(m_rows, n_cols, hw, per_crop, min_ctas=132):
    """launch_pw_tc2's column tile: narrowed (not below 48) until the grid has ``min_ctas`` CTAs (option pw_min_ctas)."""
    m_tiles = (m_rows // hw) * _cdiv(hw, 128) if per_crop else _cdiv(m_rows, 128)
    nt = _col_tile(n_cols, 128)
    while nt > 48 and m_tiles * _cdiv(n_cols, nt) < min_ctas:
        parts = _cdiv(n_cols, nt) + 1
        t = (_cdiv(n_cols, parts) + 15) & ~15
        if t >= nt:
            break
        nt = t
    return nt


def pw_tc3_taken(nb):
    """plan_pw_tc3 on block 1's project (12544 pixels, K 32, N 16): at least three 128-row tiles per CTA."""
    tpc_all = _cdiv(112 * 112, 128)
    groups = max(1, min(tpc_all, _cdiv(1536, nb)))
    return _cdiv(tpc_all, groups) >= 3


def _split(ctas, chunks):
    s = 1
    while s < chunks and ctas * s < SPLIT_CTAS:
        s += 1
    return s


def pass_route(nb, sms, prec):
    """One pass of nb crops: (features, profile layer names, launches).  A feature is what a batch-size switch selects;
    boolean features pick a kernel, integer ones partition a kernel's work (chunks per CTA, column tiles)."""
    f = {"se+head batched": nb >= 64}
    names = {"stem", "head.conv", "head.fc_decode"}
    launches = 2 + (2 if nb >= 64 else 1)          # stem, head conv, GAP + Dense/decode (two kernels from 64 crops)
    for i, b in BLOCKS.items():
        hw = b.hout * b.hout
        se = True
        expand_on_tc2 = False
        if prec == "fp32":
            kinds = (["expand"] if b.has_expand else []) + ["dw"]
        elif i == 1:
            kinds = ["dw"]
            if prec == "bf16":
                f["b01 KD split"] = _split(nb, B1_KD_TILES)
        elif prec == "bf16" and i >= 7:
            split = _split(nb, KD_CHUNKS[i])
            f["b%02d KD expand on chip" % i] = split == 1
            f["b%02d KD split" % i] = split
            kinds = (["expand"] if split > 1 else []) + ["kd"]
            expand_on_tc2 = split > 1
        else:
            tiles, per_cta, chunks = K1_PLAN[i]
            split = _split(tiles * _cdiv(nb, per_cta), chunks)
            f["b%02d K1 chunks per CTA" % i] = _cdiv(chunks, split)
            if prec == "bf16" and i in K1X_BLOCKS:
                f["b%02d K1X" % i] = split == 1
            if tiles == 1 and split == 1:
                se = False                          # SE tail: the K1 CTA gates its own output in place
                f["b%02d K1 SE tail" % i] = True
            elif tiles == 1:
                f["b%02d K1 SE tail" % i] = False
            kinds = ["k1"]
        if se:
            kinds.append("se")
        kinds.append("project")
        names |= {"b%02d.%s" % (i, k) for k in kinds}
        launches += len(kinds)
        if prec == "fp32":
            continue
        if expand_on_tc2:
            f["b%02d expand column tile" % i] = pw_tc2_tile(nb * b.hin * b.hin, b.cexp, b.hin * b.hin, False)
        # the project: K2 if ungated or on a small map and with two tiles per SM; else pw_tc3 (block 1) or pw_tc2
        if not se or hw <= 196:
            on_k2 = k2_tiles(nb * hw, b.cout) >= 2 * sms
            f["b%02d project on K2" % i] = on_k2
        else:
            on_k2 = False
        if i == 1:
            f["b01 project on pw_tc3"] = pw3 = pw_tc3_taken(nb)
            if pw3:
                continue
        if not on_k2:
            f["b%02d project column tile" % i] = pw_tc2_tile(nb * hw, b.cout, hw, se and hw >= 784)
    if prec != "fp32":
        f["head conv on K2"] = k2_tiles(nb * 49, 1280) >= 2 * sms
    return f, names, launches


def passes(n, streams=2, chunk=MAX_N, graph=False):
    """(offset, crops) of the passes of a device-resident n-crop call, and whether they run on two streams."""
    if streams >= 2 and not graph and 64 <= n <= chunk:
        per = (n + 1) // 2
        return [(0, per), (per, n - per)], True
    return [(o, min(chunk, n - o)) for o in range(0, n, chunk)], False


def routes(n, sms, prec, streams=2, chunk=MAX_N):
    """What a profiled forward of n crops shows: profile layer names and launch count, with the features of each pass."""
    ps, two = passes(n, streams, chunk)
    feats, names, launches = [], set(), 0
    for _off, nb in ps:
        f, nm, la = pass_route(nb, sms, prec)
        feats.append(f)
        names |= nm
        launches += la
    return dict(passes=ps, two_streams=two, features=feats, names=names, launches=launches)


def switches(sms, prec, streams=2, kernels_only=False):
    """Every n in 2..MAX_N whose route differs from n - 1's, with what changed: [(n, [feature, ...])].  A two-stream
    switch is crossed once per half, so it appears at two neighbouring n.  ``kernels_only``: boolean features only."""
    out = []
    prev = routes(1, sms, prec, streams)
    for n in range(2, MAX_N + 1):
        cur = routes(n, sms, prec, streams)
        what = ["two streams"] if cur["two_streams"] != prev["two_streams"] else []
        if not what:
            for h, (fa, fb) in enumerate(zip(prev["features"], cur["features"])):
                what += ["%s%s" % (k, " (half %d)" % h if cur["two_streams"] else "") for k in sorted(fb)
                         if fa.get(k) != fb[k] and (isinstance(fb[k], bool) or not kernels_only)]
        if what:
            out.append((n, what))
        prev = cur
    return out


def sweep_sizes(sms, prec, streams, full):
    """All of 1..MAX_N, or 1..160 plus +-3 around every predicted switch up to MAX_N, plus MAX_N - 7..MAX_N."""
    if full:
        return list(range(1, MAX_N + 1))
    ns = set(range(1, 161)) | set(range(MAX_N - 7, MAX_N + 1))
    for n, _what in switches(sms, prec, streams):
        ns |= {v for v in range(n - 3, n + 4) if 1 <= v <= MAX_N}
    return sorted(ns)


# ----------------------------------------------------------------------------- bitwise comparison
def mismatches(ref_ang, ref_lg, idx, ang, lg):
    """Positions whose angles or logits differ in any bit from their crop's reference (idx: pool crop per position)."""
    ra = np.ascontiguousarray(ref_ang[idx], np.float32).view(np.uint32)
    rl = np.ascontiguousarray(ref_lg[idx], np.float32).view(np.uint32)
    ga = np.ascontiguousarray(ang, np.float32).view(np.uint32)
    gl = np.ascontiguousarray(lg, np.float32).view(np.uint32)
    return np.flatnonzero((ra != ga).any(axis=1) | (rl != gl).any(axis=1))


def test_mismatch_reports_one_ulp():
    """Negative control on the host: a one-ulp change of one logit, and a sign of zero, are reported."""
    rng = np.random.default_rng(3)
    ref_ang = rng.normal(size=(POOL, 3)).astype(np.float32)
    ref_lg = rng.normal(size=(POOL, 252)).astype(np.float32)
    idx = rng.permutation(POOL)[:20]
    ang, lg = ref_ang[idx].copy(), ref_lg[idx].copy()
    assert mismatches(ref_ang, ref_lg, idx, ang, lg).size == 0
    lg[7, 131] = np.nextafter(lg[7, 131], np.float32(np.inf))
    assert mismatches(ref_ang, ref_lg, idx, ang, lg).tolist() == [7]
    lg[7, 131] = ref_lg[idx[7], 131]
    ref_ang[idx[13], 2] = 0.0
    ang[13, 2] = -0.0
    assert mismatches(ref_ang, ref_lg, idx, ang, lg).tolist() == [13]


def test_route_model_plans():
    """The model's plan tables against the planners themselves (tools/route_plan_dump.cu, tools/k1_plan_dump.cu), and its
    switch list at 132 and 114 SMs pinned."""
    exe_dir = os.path.join(ROOT, "build_tmp")
    os.makedirs(exe_dir, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    out = {}
    for tool in ("route_plan_dump", "k1_plan_dump"):
        exe = os.path.join(exe_dir, tool + "_sweep")
        r = subprocess.run([nvcc, "-std=c++17", "-arch=sm_90a", "-o", exe, os.path.join(ROOT, "tools", tool + ".cu")],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out[tool] = exe
    for crops in (1, 8, 17, 33, 34, 85, 86, 120, 135, 136, 227, 228, 256):
        txt = subprocess.run([out["route_plan_dump"], str(crops)], capture_output=True, text=True, check=True).stdout
        seen = 0
        for m in re.finditer(r"k2 \w+\s+b(\d+) M (\d+) K (\d+) N (\d+) gate \d : n_tile (\d+) n_tiles (\d+) tiles (\d+)", txt):
            M, N, tiles = int(m.group(2)), int(m.group(4)), int(m.group(7))
            assert k2_tiles(M, N) == tiles and _col_tile(N, 64) == int(m.group(5)), m.group(0)
            seen += 1
        assert seen == 13                               # expand and project of six late-block shapes, head conv
        for m in re.finditer(r"kd b(\d+) cc \d+ threads \d+ strips \d+ pw \d+ smem \d+ chunks (\d+)", txt):
            if int(m.group(1)) >= 7:
                assert KD_CHUNKS[int(m.group(1))] == int(m.group(2)), m.group(0)
        pw3 = re.search(r"pw3 b01 tiles_per_crop \d+ tpc (\d+)", txt)
        assert (pw3 is not None) == pw_tc3_taken(crops), crops
    txt = subprocess.run([out["k1_plan_dump"]], capture_output=True, text=True, check=True).stdout
    rows = re.findall(r"b(\d+) +\d+-> ?\d+ .*: +(\d+)x(\d+) +r\d cc\d+ +nt\d+ nb(\d) .* chunks +(\d+)", txt)
    assert len(rows) == 11, txt
    for idx, th, tw, nbc, chunks in rows:
        b = BLOCKS[int(idx)]
        assert K1_PLAN[int(idx)] == ((b.hout // int(th)) * (b.hout // int(tw)), int(nbc), int(chunks)), idx
    # the kernel switches of the default bf16 route (both halves of a two-stream switch)
    got = {sms: [n for n, _w in switches(sms, "bf16", kernels_only=True)] for sms in (132, 114)}
    assert got[132] == [3, 8, 30, 32, 34, 64, 67, 68, 127, 128, 171, 172, 239, 240, 271, 272, 455, 456], got[132]
    assert got[114] == [3, 8, 29, 30, 32, 64, 127, 128, 147, 148, 235, 236, 239, 240, 391, 392], got[114]
    fp16 = [n for n, _w in switches(132, "fp16", kernels_only=True)]
    assert fp16 == [32, 34, 64, 67, 68, 127, 128, 171, 172, 239, 240, 271, 272, 455, 456, 477, 478], fp16
    assert [n for n, _w in switches(132, "fp32", kernels_only=True)] == [64, 127, 128]


# ----------------------------------------------------------------------------- GPU: pool, references, sweep
def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def make_pool():
    """48 distinct crops: the 2 Sample and 6 jitter crops, all 0, all 255, a 0/255 checkerboard, four gradients and
    uniform random crops."""
    s = np.load(os.path.join(GOLD, "sample_crops.npy"))
    j = np.load(os.path.join(GOLD, "jitter_crops.npy"))
    yy, xx = np.mgrid[0:224, 0:224]
    cb = np.repeat((((yy + xx) % 2) * 255).astype(np.uint8)[..., None], 3, axis=2)
    ramp = (np.arange(224) * 255 // 223).astype(np.uint8)
    grads = [np.broadcast_to(ramp[None, :, None], (224, 224, 3)), np.broadcast_to(ramp[:, None, None], (224, 224, 3)),
             ((yy + xx) * 255 // 446).astype(np.uint8)[..., None].repeat(3, axis=2),
             np.stack([ramp[None, :].repeat(224, 0), ramp[:, None].repeat(224, 1), 255 - ramp[None, :].repeat(224, 0)], axis=2)]
    fixed = np.concatenate([s, j, np.zeros((1, 224, 224, 3), np.uint8), np.full((1, 224, 224, 3), 255, np.uint8), cb[None],
                            np.stack(grads)])
    rnd = np.random.default_rng(4242).integers(0, 256, (POOL - len(fixed), 224, 224, 3), dtype=np.uint8)
    pool = np.ascontiguousarray(np.concatenate([fixed, rnd]))
    assert pool.shape == (POOL, 224, 224, 3) and len({p.tobytes() for p in pool}) == POOL
    return pool


def positions(n):
    """The seeded pool crop at each of n positions: permutations of the pool laid end to end."""
    rng = np.random.default_rng(n)
    return np.concatenate([rng.permutation(POOL) for _ in range(_cdiv(n, POOL))])[:n]


def _model(prec, opts, max_batch, streams=2, chunk=None):
    import whenet_b200
    m = whenet_b200.WHENet(SNAP, device=0, precision=prec, max_batch=max_batch)
    m.set_option("chunk", chunk or max_batch)
    m.set_option("fused", 1)
    m.set_option("streams", streams)
    for k, v in opts.items():
        m.set_option(k, v)
    return m


class Dev:
    """The pool on the device once, and input / output buffers for up to MAX_N crops gathered from it."""

    def __init__(self, pool):
        import torch
        self.torch = torch
        self.pool = torch.from_numpy(pool).cuda()
        self.x = torch.empty((MAX_N, 224, 224, 3), dtype=torch.uint8, device="cuda")
        self.ang = torch.empty((MAX_N, 3), dtype=torch.float32, device="cuda")
        self.lg = torch.empty((MAX_N, 252), dtype=torch.float32, device="cuda")

    def gather(self, idx):
        t = self.torch
        n = len(idx)
        t.index_select(self.pool, 0, t.from_numpy(np.asarray(idx, np.int64)).cuda(), out=self.x[:n])
        t.cuda.synchronize()                    # the forward runs on the context's own stream
        return self.x[:n]

    def forward(self, m, idx, profile=False):
        """Device-resident forward of the pool crops idx: (angles, logits, launches, profile names or None)."""
        n = len(idx)
        x = self.gather(idx)
        self.ang[:n].fill_(np.nan)
        self.lg[:n].fill_(np.nan)
        self.torch.cuda.synchronize()
        l0 = m.launch_count()
        m.forward_device(x, self.ang[:n], self.lg[:n])
        m.synchronize()
        out = (self.ang[:n].cpu().numpy(), self.lg[:n].cpu().numpy(), m.launch_count() - l0)
        names = None
        if profile:
            m.enable_profile(True)
            m.forward_device(x, self.ang[:n], self.lg[:n])
            m.synchronize()
            names = {p["name"] for p in m.read_profile()}
            m.enable_profile(False)
        return out + (names,)


_STATE = {}


def _dev():
    if "dev" not in _STATE:
        _STATE["pool"] = make_pool()
        _STATE["dev"] = Dev(_STATE["pool"])
    return _STATE["dev"]


def references(prec, opts):
    """Every pool crop's angles and logits from a fresh context at n = 8 on one stream."""
    key = (prec, tuple(sorted(opts.items())))
    if key not in _STATE:
        dev = _dev()
        m = _model(prec, opts, 8, streams=1)
        try:
            out = [dev.forward(m, list(range(o, o + 8)))[:2] for o in range(0, POOL, 8)]
        finally:
            m.close()
        _STATE[key] = (np.concatenate([a for a, _ in out]), np.concatenate([lg for _, lg in out]))
    return _STATE[key]


def _oracle_angles(oracle64):
    if "oracle" not in _STATE:
        _dev()
        _STATE["oracle"] = np.stack(oracle64.get_angle(_STATE["pool"]), axis=1).astype(np.float64)
    return _STATE["oracle"]


def _report(bad, limit=12):
    return "; ".join("n=%d: %d positions differ, first %s" % (n, len(p), [(int(q), int(c)) for q, c in p[:3]])
                     for n, p in bad[:limit])


@gpu
@pytest.mark.parametrize("route", list(ROUTES))
def test_pool_references_match_oracle(route, oracle64):
    """The n = 8 references of the pool crops against float64: within the route's parity tolerance (DESIGN §2) for the
    Sample, jitter and uniform random crops, and for every crop in fp32.  The 16-bit tolerances are stated for natural and
    random crops; the synthetic crops (constant, checkerboard, gradients) are checked element by element at every stage
    instead, within 2 B of float64 on the stage's own GPU input."""
    prec, opts, _s = ROUTES[route]
    ang, lg = references(prec, opts)
    ref = _oracle_angles(oracle64)
    assert np.isfinite(ang).all() and np.isfinite(lg).all()
    d = np.abs(ang.astype(np.float64) - ref)
    d = np.minimum(d, 360 - d).max(axis=1)
    documented = [i for i in range(POOL) if prec == "fp32" or i not in SYNTHETIC]
    print("%s: max |angle - oracle64|: %.4f deg over the Sample, jitter and random crops, %s deg on the synthetic crops %s" %
          (route, d[[i for i in range(POOL) if i not in SYNTHETIC]].max(), d[SYNTHETIC].round(4).tolist(), SYNTHETIC))
    assert d[documented].max() <= TOL[prec], (route, d.round(4).tolist())
    if route in ("bf16", "fp16"):
        _taps, stats = _n8_taps(prec, opts, SYNTHETIC, oracle64)
        print("%s synthetic crops: worst |got - ref| / B %s" % (route, {k: round(v[0], 3) for k, v in stats.items() if not k.startswith("_")}))


@gpu
@pytest.mark.parametrize("route", list(ROUTES))
def test_batch_sweep_bitwise(route):
    """Every swept n: every position bit-identical to its crop's n = 8 reference, launch count and profile layer names as
    the route model predicts, and both sides of every predicted switch swept.  The bf16 route then reruns n = 1, 239 and
    512 on the same context, whose tensor-map caches the sweep has cleared several times."""
    prec, opts, streams = ROUTES[route]
    full = route == "bf16"
    sms = _sms()
    dev = _dev()
    ref_ang, ref_lg = references(prec, opts)
    ns = sweep_sizes(sms, prec, streams, full)
    sw = switches(sms, prec, streams)
    swept = set(ns)
    missing = [n for n, _w in sw if not {n - 1, n} <= swept]
    assert not missing, (route, missing)
    m = _model(prec, opts, MAX_N, streams)
    bad, model_bad, forwards = [], [], 0
    t0 = time.time()
    try:
        for n in ns:
            idx = positions(n)
            ang, lg, launches, names = dev.forward(m, idx, profile=True)
            forwards += 2
            p = mismatches(ref_ang, ref_lg, idx, ang, lg)
            if p.size:
                bad.append((n, list(zip(p, idx[p]))))
            r = routes(n, sms, prec, streams)
            if launches != r["launches"] or names != r["names"]:
                model_bad.append((n, launches, r["launches"], sorted(names ^ r["names"])))
        if full:
            for n in (1, 239, 512):
                idx = positions(n)
                ang, lg, _l, _n = dev.forward(m, idx)
                forwards += 1
                p = mismatches(ref_ang, ref_lg, idx, ang, lg)
                if p.size:
                    bad.append((n, list(zip(p, idx[p]))))
    finally:
        m.close()
    wall = time.time() - t0
    print("MEASURED batch sweep %s (%s, %d SMs): n %d..%d, %d batch sizes, %d forwards, %d switches crossed from both sides "
          "at n = %s, %.1f s" % (route, prec, sms, ns[0], ns[-1], len(ns), forwards, len(sw), [n for n, _w in sw], wall))
    for n, what in switches(sms, prec, streams, kernels_only=True):
        print("  switch at n=%d: %s" % (n, ", ".join(what)))
    assert not model_bad, (route, model_bad[:8])
    assert not bad, (route, _report(bad))


def _tap_sizes(sms, prec):
    """Both sides of every kernel switch of the two-stream route, and the largest batch."""
    ns = set()
    for n, _w in switches(sms, prec, 2, kernels_only=True):
        ns |= {n - 1, n}
    return sorted(ns | {MAX_N})


def _n8_taps(prec, opts, crops, oracle64):
    """Faithful taps of the pool crops ``crops`` (at most 8) from a fresh n = 8 context on one stream, checked once against
    float64 element by element (every stage within 2 B, elementwise_check)."""
    key = ("taps", prec, tuple(crops))
    if key in _STATE:
        return _STATE[key]
    dev = _dev()
    ref_ang, ref_lg = references(prec, opts)
    idx = list(crops) + [i for i in range(POOL) if i not in crops][:8 - len(crops)]
    m = _model(prec, opts, 8, streams=1)
    try:
        m.enable_taps(True, faithful=True, crops=list(range(len(crops))))
        ang, lg, _l, _n = dev.forward(m, idx)
        taps = ec.read_taps(m, len(crops))
    finally:
        m.close()
    assert mismatches(ref_ang, ref_lg, np.asarray(idx), ang, lg).size == 0, "taps changed the n = 8 results"
    a = wb.BF16 if prec == "bf16" else wb.FP16

    def get(name):
        v = taps.get(name)
        return None if v is None else v.reshape(-1)
    stats = ec.check_stages("n8_%s_crops%s" % (prec, list(crops)), get, _STATE["pool"][list(crops)], ang[:len(crops)], a,
                            oracle64, oracle64.stage_layers()["blocks"], {})
    _STATE[key] = (taps, stats)
    return _STATE[key]


@gpu
@pytest.mark.parametrize("route", ["bf16", "fp16"])
def test_taps_at_switches(route, oracle64):
    """At both sides of every kernel switch, faithful taps of up to four edge crops (the last crop of each half, the last
    ragged group of four, a crop sharing a K2 row tile) are bit-identical to the same crop's n = 8 taps, where the crops at
    those positions are the TAP_POOL crops.  The n = 8 taps themselves are within 2 B of float64 (elementwise_check)."""
    prec, opts, streams = ROUTES[route]
    sms = _sms()
    dev = _dev()
    ref_ang, ref_lg = references(prec, opts)
    ref_taps, stats = _n8_taps(prec, opts, TAP_POOL, oracle64)
    store = wb.BF16.store if prec == "bf16" else wb.FP16.store
    m = _model(prec, opts, MAX_N, streams)
    bad, t0, ns = [], time.time(), _tap_sizes(sms, prec)
    try:
        for n in ns:
            r = routes(n, sms, prec, streams)
            edges = ec.edge_crops(r["passes"], sms, prec == "bf16")
            sel = [c for k, c in edges if k == "last"] + [c for k, c in edges if k == "ragged"][-1:] + \
                  [c for k, c in edges if k == "k2_shared"]
            sel = list(dict.fromkeys(sel))[:len(TAP_POOL)]
            idx = positions(n)
            for j, c in enumerate(sel):
                idx[c] = TAP_POOL[j]
            for off, nb in r["passes"]:
                # one tapped forward per pass: its halves may differ in which blocks gate in place, and one dw tap
                # holds one form
                rows = [j for j, c in enumerate(sel) if off <= c < off + nb]
                if not rows:
                    continue
                m.enable_taps(True, faithful=True, crops=[sel[j] for j in rows])
                ang, lg, _l, _n = dev.forward(m, idx)
                p = mismatches(ref_ang, ref_lg, idx, ang, lg)
                if p.size:
                    bad.append((n, "positions %s" % p[:4].tolist()))
                big = ec.read_taps(m, len(rows))
                small = {k: v[rows] for k, v in ref_taps.items()}
                d = ec.taps_mismatch(big, small, store)
                if d:
                    bad.append((n, "crops %s taps %s" % ([sel[j] for j in rows], d)))
    finally:
        m.close()
    print("MEASURED taps at switches %s: %d batch sizes %s, %.1f s; n = 8 taps within %s of 2 B" %
          (route, len(ns), ns, time.time() - t0, {k: round(v[0], 3) for k, v in stats.items() if not k.startswith("_")}))
    assert not bad, (route, bad[:8])


@gpu
def test_host_and_chunked_paths_bitwise():
    """get_angle / _forward on pageable numpy and forward_host on pinned buffers, Python chunking past max_batch and ragged
    single-stream passes: the same bits as the device sweep's references."""
    import torch
    _dev()
    pool = _STATE["pool"]
    ref_ang, ref_lg = references("bf16", {})
    bad = []
    m = _model("bf16", {}, MAX_N)
    try:
        for n in (55, 56, 57, 63, 64, 65, 110, 111, 112, 127, 128, 239, 240, 511, 512):
            idx = positions(n)
            x = np.ascontiguousarray(pool[idx])
            ang, lg = m._forward(x, want_logits=True)              # get_angle's path: pageable input, staged upload
            yaw, pitch, roll = m.get_angle(x)
            if mismatches(ref_ang, ref_lg, idx, ang, lg).size or not np.array_equal(np.stack([yaw, pitch, roll], 1), ang):
                bad.append(("pageable", n))
            xp = torch.from_numpy(x).pin_memory()
            ap = torch.empty((n, 3), dtype=torch.float32).pin_memory()
            lp = torch.empty((n, 252), dtype=torch.float32).pin_memory()
            m.forward_host(xp, ap, lp)
            if mismatches(ref_ang, ref_lg, idx, ap.numpy(), lp.numpy()).size:
                bad.append(("pinned", n))
    finally:
        m.close()
    m = _model("bf16", {}, 77)                                     # batches past max_batch: chunked in Python
    try:
        for n in (76, 77, 78, 154, 155):
            idx = positions(n)
            ang, lg = m._forward(np.ascontiguousarray(pool[idx]), want_logits=True)
            if mismatches(ref_ang, ref_lg, idx, ang, lg).size:
                bad.append(("max_batch 77", n))
    finally:
        m.close()
    m = _model("bf16", {}, MAX_N, chunk=100)                      # passes of 100, 100 and 50 crops on one stream
    try:
        idx = positions(250)
        ang, lg, launches, _n = _dev().forward(m, idx)
        if mismatches(ref_ang, ref_lg, idx, ang, lg).size:
            bad.append(("chunk 100", 250))
        assert launches == sum(pass_route(nb, _sms(), "bf16")[2] for nb in (100, 100, 50))
    finally:
        m.close()
    assert not bad, bad


@gpu
def test_graph_cache_eviction_bitwise():
    """With graph replay on, more than 8 distinct batch sizes evict the first graphs; replaying those again (recaptured)
    and the cached ones gives the same bits."""
    dev = _dev()
    ref_ang, ref_lg = references("bf16", {})
    ns = [1, 5, 17, 33, 64, 65, 100, 127, 128, 200, 333]
    bad = []
    m = _model("bf16", {"graph": 1}, MAX_N)
    try:
        for n in ns + ns[:3] + ns[-3:] + ns[:3]:
            idx = positions(n)
            ang, lg, launches, _n = dev.forward(m, idx)
            if mismatches(ref_ang, ref_lg, idx, ang, lg).size:
                bad.append(n)
            assert launches == routes(n, _sms(), "bf16", streams=1)["launches"], n
    finally:
        m.close()
    assert not bad, bad


@gpu
def test_sweep_reports_other_rounding():
    """Negative control: references taken with pw_variant = 3 (K2 on every project, which rounds a*g instead of w*g on
    blocks 1-5) are reported as mismatches by the default bf16 forward."""
    dev = _dev()
    ref_ang, ref_lg = references("bf16", {"pw_variant": 3})
    m = _model("bf16", {}, MAX_N)
    out = {}
    try:
        for n in (8, 239, 512):
            idx = positions(n)
            ang, lg, _l, _n = dev.forward(m, idx)
            out[n] = mismatches(ref_ang, ref_lg, idx, ang, lg).size / n
    finally:
        m.close()
    print("MEASURED negative control pw_variant=3 references: share of positions reported %s" % out)
    assert all(v > 0.5 for v in out.values()), out
