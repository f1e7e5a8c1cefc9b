"""Every WHENet stage of a tapped forward against float64 on its own GPU input (DESIGN §2.1), the checker shared by
test_gpu_block_elementwise.py (8 crops, every block route) and test_gpu_throughput_elementwise.py (selected crops of the
throughput batches).

A stage's input is the previous tap (an exact float32 copy of the storage type), so |got - ref| <= 2 B must hold for every
element, B being the first-order bound of tests/whenet_bounds.py.  Every stage reference is per crop, so the taps of any
subset of a batch's crops can be checked on their own.
"""
import numpy as np

import whenet_bounds as wb
from whenet_oracle import preprocess, softmax

KINDS = ["stem", "dw", "dwg", "gate", "block", "head", "pooled", "angles"]


def bf16(x):
    import torch
    return torch.from_numpy(np.asarray(x, dtype=np.float64)).to(torch.bfloat16).to(torch.float64).numpy()


def f32(x):
    return np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)


def round16(x, store):
    """Round-to-nearest-even to the 16-bit storage type."""
    return bf16(x) if store == "bf16" else np.asarray(x, dtype=np.float64).astype(np.float16).astype(np.float64)


def tap_reader(m):
    """m.tap, with None for a tap the last forward did not write."""
    from whenet_b200 import WhenetError

    def get(name):
        try:
            return m.tap(name)
        except WhenetError:
            return None
    return get


TAP_NAMES = ["stem", "head", "pooled"] + ["%s%d" % (k, i) for i in range(1, 17) for k in ("dw", "dwg", "gate", "block")]


def read_taps(m, k):
    """Every tap the last forward of m wrote, as (k crops, elements per crop)."""
    get = tap_reader(m)
    out = {}
    for name in TAP_NAMES:
        v = get(name)
        if v is not None:
            out[name] = v.reshape(k, -1)
    return out


def check(route, kind, name, got, ref, b, shape, store, stats):
    got = got.reshape(shape).astype(np.float64)
    assert np.isfinite(got).all(), (route, name, "non-finite values")
    err = np.abs(got - ref)
    r = err / b
    i = np.unravel_index(int(np.argmax(r)), r.shape)
    assert r[i] <= 2.0, ("%s %s: element %s got %.9g ref %.9g B %.3g (ratio %.2f)" %
                         (route, name, tuple(int(v) for v in i), got[i], ref[i], b[i], r[i]))
    prev = stats.setdefault(kind, (0.0, ""))
    if r[i] > prev[0]:
        stats[kind] = (float(r[i]), name)
    if store is not None:
        stats["_n"] = stats.get("_n", 0) + err.size
        stats["_in"] = stats.get("_in", 0) + int((err <= wb.ulp(ref, store)).sum())
    return got


def project_forms(oracle, b, d, g, res):
    """The GPU's bf16 project outputs as each gate rounding gives them (fp32 accumulation and epilogue emulated; the few
    elements whose accumulation order flips a rounding do not match either way)."""
    k, sh = oracle._fold(b["proj"], b["proj_bn"])
    wq = bf16(k[0, 0])
    n, c = d.shape[0], d.shape[3]
    acc = {"w*g": np.einsum("npk,nkj->npj", d.reshape(n, -1, c), bf16(wq[None] * g[:, :, None])),
           "a*g": bf16(d * g[:, None, None, :]).reshape(n, -1, c) @ wq}
    out = {}
    for form, v in acc.items():
        y = f32(f32(v.reshape(d.shape[:3] + (wq.shape[1],))) + f32(sh))
        out[form] = bf16(f32(y + res) if res is not None else y)
    return out


def decode64(logits):
    out = []
    for lg, off in zip(logits, (180.0, 99.0, 99.0)):
        v = np.arange(lg.shape[1], dtype=np.float64)
        out.append((softmax(lg) * v).sum(axis=1) * 3 - off)
    return out


def check_stages(route, get, x, ang, a, oracle, blocks, stats, keep=None, project_form=None):
    """Every tap of the crops x (in tap-row order) against float64 on its GPU input.  ``get(name)``: the flat float32 tap
    or None; ``ang``: the forward's (n, 3) angles of the same crops.  A block gated in place has "dwg%d" (the stored
    d * g) instead of "dw%d": its gate is then checked on d recovered as dwg / g, and its project as an ungated conv of
    dwg.  ``keep``: dict that receives every block's references (the negative controls); ``project_form``: the gate
    rounding ("w*g" or "a*g") the bf16 projects of blocks 1-5 must show."""
    nb = len(x)
    xn = preprocess(x)
    r = oracle.run_stage("stem", xn)
    stem = get("stem").reshape(r["out"].shape).astype(np.float64)
    if a.stem_store == "fp16" and a.store == "bf16":
        assert np.array_equal(stem.astype(np.float16).astype(np.float64), stem), "stem tap is not fp16"
    check(route, "stem", "stem", stem, r["out"], wb.stem(r, a), r["out"].shape, a.stem_store, stats)
    if keep is not None:
        keep["stem"] = (stem, r)
    prev = stem
    for i in range(1, 17):
        b = blocks[i - 1]
        rd = oracle.run_stage("dw", prev, i)
        b_e = wb.expand(rd, a, prev.shape[-1]) if b["expand"] is not None else None
        bd = wb.depthwise(rd, a, i, b["stride"], b_e)
        dw, dwg = get("dw%d" % i), get("dwg%d" % i)
        assert (dw is None) != (dwg is None), (route, i, "exactly one of dw / dwg must be tapped")
        hw = rd["out"].shape[1] * rd["out"].shape[2]
        res = prev if b["skip"] else None
        if dw is not None:
            d = check(route, "dw", "dw%d" % i, dw, rd["out"], bd, rd["out"].shape, a.store, stats)
            rg = oracle.run_stage("gate", d, i)
            g = check(route, "gate", "gate%d" % i, get("gate%d" % i), rg["out"], wb.gate(rg, a, np.abs(d).mean(axis=(1, 2)), hw),
                      rg["out"].shape, None, stats)
            rp = oracle.run_stage("project", d, i, gate=g, resid=res)
        else:
            dg = dwg.reshape(rd["out"].shape).astype(np.float64)
            assert np.isfinite(dg).all(), (route, "dwg%d" % i, "non-finite values")
            gt = get("gate%d" % i).reshape(nb, -1).astype(np.float64)
            assert np.isfinite(gt).all(), (route, "gate%d" % i, "non-finite values")
            # The stored d the gate was computed from is gone: dwg / g gives it back within a 16-bit rounding of the product,
            # and the squeeze summed fp32 values one store rounding from it (2 u_store |d|).  Where g is 0 the product
            # carries no d: the reference d stands in, within its own bound.
            pos = gt[:, None, None, :] > 0
            with np.errstate(divide="ignore", invalid="ignore"):
                d_est = np.where(pos, dg / np.where(pos, gt[:, None, None, :], 1.0), rd["out"])
            b_in = np.where(pos, (2 * wb.U[a.store] + wb.U32) * np.abs(d_est), bd).mean(axis=(1, 2))
            rg = oracle.run_stage("gate", d_est, i)
            bg = wb.gate(rg, a, np.abs(d_est).mean(axis=(1, 2)), hw, b_in_mean=b_in)
            g = check(route, "gate", "gate%d" % i, gt, rg["out"], bg, rg["out"].shape, None, stats)
            ref = rd["out"] * rg["out"][:, None, None, :]
            d = check(route, "dwg", "dwg%d" % i, dg, ref, wb.gated(bd, rd["out"], rg["out"], bg, a), ref.shape, a.store, stats)
            rp = oracle.run_stage("project", d, i, gate=np.ones_like(g), resid=res)
        y = check(route, "block", "block%d" % i, get("block%d" % i), rp["out"], wb.project(rp, a, d.shape[-1]),
                  rp["out"].shape, a.store, stats)
        if project_form is not None and i <= 5:
            forms = project_forms(oracle, b, d, g, res)
            share = {f: float((v == y).mean()) for f, v in forms.items()}
            other = "a*g" if project_form == "w*g" else "w*g"
            print("%s block %d project: bitwise share %s" % (route, i, share))
            assert share[project_form] >= 0.9 and share[project_form] > share[other] + 0.05, (route, i, share)
        if keep is not None:
            keep[i] = (prev, rd, bd, d, rg, g, rp, y)
        prev = y
    rh = oracle.run_stage("head", prev)
    h = check(route, "head", "head", get("head"), rh["out"], wb.head(rh, a), rh["out"].shape, a.store, stats)
    p = check(route, "pooled", "pooled", get("pooled"), h.mean(axis=(1, 2)), wb.pooled(h), (nb, 1280), None, stats)
    rdn = oracle.run_stage("dense", p)
    ref_ang = np.stack([v.astype(np.float64) for v in decode64(rdn["logits"])], axis=1)
    check(route, "angles", "angles", np.asarray(ang, dtype=np.float64), ref_ang, np.stack(wb.angles(rdn, rdn["logits"]), axis=1),
          (nb, 3), None, stats)
    stats["_ulp"] = stats["_in"] / stats["_n"]
    print("%s: worst ratio %s; %.4f of stored elements within one ulp" %
          (route, {k: "%.3f (%s)" % v for k, v in stats.items() if not k.startswith("_")}, stats["_ulp"]))
    return stats


# K1X instances (bf16): output tiles per crop and resident CTAs per SM, as in test_gpu_k1x_persistent.py
K1X_TILES = {2: 49, 3: 16, 4: 16, 6: 4}
K1X_CTAS_PER_SM = {2: 3, 3: 3, 4: 3, 6: 2}
MAX_SEL = 16


def halves(n):
    """(offset, crops) of the two half batches of a two-stream pass."""
    per = (n + 1) // 2
    return [(0, per), (per, n - per)]


def edge_crops(passes, sms, k1x):
    """(kind, crop) at the schedule's edges of the given passes ((offset, crops) each), in priority order: "first" / "last"
    crop of each pass, the last (ragged) group of four of se_gate_batch / head_fc_decode_batch ("ragged"), a crop sharing a
    128-row K2 tile with its neighbour at 196 and 49 pixels per crop ("k2_shared"), and (bf16, k1x) the crop holding the
    first item of each K1X block's second persistent round ("k1x_round")."""
    out = []
    for off, h in passes:
        out += [("first", off), ("last", off + h - 1)]
    for off, h in passes:
        out.append(("ragged", off + (h - 1) // 4 * 4))
    off0, h0 = passes[0]
    for hw in (196, 49):
        c = next((c for c in range(h0) if (c * hw) // 128 != ((c + 1) * hw - 1) // 128), None)
        if c is not None:
            out.append(("k2_shared", off0 + c))
    if k1x:
        for b, t in K1X_TILES.items():                        # items run crop-major: the crop holding a round's first item
            grid = K1X_CTAS_PER_SM[b] * sms
            for off, h in passes:
                if h * t > grid:
                    out.append(("k1x_round", off + grid // t))
    return out


def select_crops(n, sms, k1x, passes=None, kinds=None, limit=MAX_SEL):
    """Distinct edge crops of an n-crop call (default: its two halves), in priority order, at most ``limit``; ``kinds``
    keeps only those kinds of edge_crops."""
    out = []
    for kind, c in edge_crops(passes or halves(n), sms, k1x):
        if (kinds is None or kind in kinds) and c not in out:
            out.append(c)
    return out[:limit]


def taps_mismatch(big, small, store):
    """Names of the taps (dict name -> (crops, elements)) that differ bit for bit between two runs of the same crops.  A block
    whose depthwise output is gated in place on one side only is compared through round16(float32(d) * float32(g)), which
    is what the in-place gate computes."""
    bad = []
    for i in range(1, 17):
        for k in ("gate", "block"):
            if not np.array_equal(big["%s%d" % (k, i)], small["%s%d" % (k, i)]):
                bad.append("%s%d" % (k, i))
        kb = "dwg%d" % i if "dwg%d" % i in big else "dw%d" % i
        ks = "dwg%d" % i if "dwg%d" % i in small else "dw%d" % i
        if kb == ks:
            ok = np.array_equal(big[kb], small[ks])
        else:
            d, dg = (small[ks], big[kb]) if kb.startswith("dwg") else (big[kb], small[ks])
            g = small["gate%d" % i]
            k_ = d.shape[0]
            emu = round16(d.reshape(k_, -1, g.shape[1]).astype(np.float32) * g.astype(np.float32)[:, None, :], store)
            ok = np.array_equal(dg, emu.reshape(k_, -1))
        if not ok:
            bad.append("%s/%s" % (kb, ks))
    for k in ("stem", "head", "pooled"):
        if not np.array_equal(big[k], small[k]):
            bad.append(k)
    return bad


def print_table(ratios, title):
    kinds = [k for k in KINDS if any(k in d for d in ratios.values())]
    print("\n" + title)
    print("%-18s" % "route" + "".join("%9s" % k for k in kinds) + "   1-ulp")
    for route, d in ratios.items():
        print("%-18s" % route + "".join("%9.3f" % d[k][0] if k in d else "%9s" % "-" for k in kinds) + "   %.4f" % d["_ulp"])
