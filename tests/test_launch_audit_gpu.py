"""Launch audit of the frame program and of the prompt / timestep refresh: every kernel launch of a real frame (contractions,
attention, GroupNorm, LayerNorm, the input heads and other small convs, upsampling, HED, the scheduler step, the u8 tail) and of
the refresh (prompt K / V^T projections, timestep embedding, time MLPs, every resnet's time bias), checked in place against a
float64 recomputation of its own inputs.  No launch is exempt: a launch without a record (kind "other") fails the audit.

StreamDiffusion.audit_step runs one frame eagerly and calls back before and after every kernel launch with the launch's record
(descriptor and plan as launched); audit_refresh does the same for the refresh.  Before: the callback snapshots everything the
launch reads (sources, weights, bias, residual, LayerNorm statistics, Q / K / V^T, normalisation inputs, the caller's u8 frame,
the whole stream-batch buffer the scheduler step rewrites in place) and the spare pitch columns of its outputs.  After: the
output is compared with the descriptor-driven reference of tests/launch_ref.py (tolerance atol * rms(ref) + rtol * |ref| per
class, bit for bit for upsample2x / maxpool2x2 / post_u8, the u8 edge map up to +-1 at float64 values within 1e-3 of an
integer), every check is shown to be discriminating by a named wrong reference that lands >= 10x the tolerance away (bit-exact
classes: differs on >= 1 % of the outputs), the spare columns must be bit-identical, and a LayerNorm-statistics producer's
fixed-point sums must match its stored fp16 rows.

The audited frame's u8 output must equal, bit for bit, a CUDA-graph step of a lane prepared identically: the audit observes
the real program.  Device memory is only ever read, never past the last row of a buffer: the spare columns of an output's last
row are not checked (the pitch can reach past the allocation when an output is a column range of a wider buffer)."""
from __future__ import annotations

import collections
import gc
import time

import pytest
import torch

from tests import launch_ref as R

pytestmark = pytest.mark.gpu

_T4 = [18, 26, 35, 45]


class _Dev:
    def __init__(self, ptr, shape, strides, typestr):
        self.__cuda_array_interface__ = {"shape": shape, "strides": strides, "typestr": typestr, "data": (ptr, False),
                                         "version": 3}


_TYPES = {torch.float16: ("<f2", 2), torch.float32: ("<f4", 4), torch.int64: ("<i8", 8), torch.uint8: ("|u1", 1)}


def _dev(ptr, rows, cols, ld, dtype=torch.float16):
    """A [rows, cols] device view with row pitch ld (elements) at ptr; never touches memory outside those elements.  (torch
    takes no read-only views: the audit only ever reads or copies them.)"""
    ts, es = _TYPES[dtype]
    return torch.as_tensor(_Dev(int(ptr), (int(rows), int(cols)), (int(ld) * es, es), ts), device="cuda")


def _snap(ptr, rows, cols, ld, dtype=torch.float16):
    if not ptr or rows <= 0 or cols <= 0:
        return None
    return _dev(ptr, rows, cols, ld, dtype).clone(memory_format=torch.contiguous_format)


def _vec(ptr, n, dtype=torch.float32):
    return _snap(ptr, 1, n, n, dtype).flatten() if ptr else None


def _spare(ptr, rows, c0, ld):
    """bits of the spare columns [c0, ld) of rows 0 .. rows-2"""
    if not ptr or rows < 2 or c0 >= ld:
        return None
    return _snap(ptr, rows - 1, ld, ld)[:, c0:].view(torch.int16)


def _src_view(v):
    rows = v["n"] * v["h"] * v["w"]
    return _snap(v["ptr"], rows, v["c"], v["ld"]).reshape(v["n"], v["h"], v["w"], v["c"])


def _kind_class(kind, d=None):
    if kind in ("igemm", "tconv"):
        if d["flags"] & R.IG_GEGLU:
            return "geglu+ln" if d["colsum"] else "geglu"
        return "contraction+ln" if d["colsum"] else "contraction"
    return {"attn": "attention", "groupnorm": "norm", "layernorm": "norm"}.get(kind, kind)


def _frac(a, b):
    """fraction of the elements where a and b differ (bit-exact classes' wrong references)"""
    return (a.to(b.device) != b).double().mean().item()


_HED = ("maxpool2x2", "hed_project", "hed_fuse")


class Auditor:
    def __init__(self):
        self.calls = 0
        self.launches = collections.Counter()     # per class
        self.checked = collections.Counter()
        self.worst = collections.defaultdict(float)
        self.worst_label = {}
        self.wrong = collections.defaultdict(collections.Counter)
        self.other = collections.Counter()
        self.labels = collections.Counter()     # (class, first word of the label)
        self.lnstat = 0.0
        self.pending = None
        self.tiles = set()        # (nb, ho, wo, tw, th, tn, swap) of every implicit-GEMM launch (not the halo-tile kernel)
        self.self_attn = set()    # (nb, sq) of every self-attention launch (K per image)
        self.stream_batch = set()  # T of every scheduler step
        # the shapes the optional branches' regimes depend on (tests/test_config_space_branches.py): "igemm" (nb, ho, wo, tw,
        # th, tn, swap, IG_SILU / IG_PAD0 flags), "conv" (kind, weight key), "d512" sq, "groupnorm" (ca, cb, hw),
        # "res_bs0" (smallconv label, nb) of a residual broadcast over the batch, "maxpool2x2" (h, w, c), "hed_fuse" (h, w)
        self.branch = collections.defaultdict(set)
        self.min_free = None       # least free HBM seen after a launch (bytes)

    def __call__(self, index, after, rec):
        from ai_rtc_agent_b200.host import capi
        kind = capi.LAUNCH_KINDS[rec.kind]
        label = rec.label.decode()
        if kind == "other":
            if not after:
                self.calls += 1
                self.other[label.split(" ")[0]] += 1
            return
        if not after:
            self.calls += 1
            self.pending = (index, getattr(self, "_before_" + ("igemm" if kind == "tconv" else kind))(rec))
        else:
            assert self.pending and self.pending[0] == index
            getattr(self, "_after_" + ("igemm" if kind == "tconv" else kind))(rec, kind, label, self.pending[1])
            self.pending = None
        torch.cuda.synchronize()
        if after:
            free = torch.cuda.mem_get_info()[0]
            self.min_free = free if self.min_free is None else min(self.min_free, free)

    def _record(self, cls, label, units, wrongs, exact=False):
        """units: error in tolerance units (bit-exact classes: 0, or inf on any difference); wrongs: name -> the wrong
        reference's distance in tolerance units (bit-exact classes: the fraction of outputs where it differs)."""
        self.launches[cls] += 1
        self.labels[cls, label.split(" ")[0]] += 1
        need = 0.01 if exact else 10.0
        assert units <= 1.0, f"{label}: error {units:.3g}x the {cls} tolerance {R.TOL.get(cls, 'bit-exact')}"
        best = max(wrongs.values()) if wrongs else 0.0
        assert wrongs and best >= need, f"{label}: no wrong reference lands far enough away ({need}: {wrongs})"
        for name, m in wrongs.items():
            if m >= need:
                self.wrong[cls][name] += 1
        self.checked[cls] += 1
        if units >= self.worst[cls]:
            self.worst[cls], self.worst_label[cls] = units, label

    # ---- contractions (igemm, tconv) ------------------------------------------------------------------------------------
    def _before_igemm(self, rec):
        d = R.as_dict(rec.igemm)
        rows, ng = R.rows_of(d), R.n_gemm(d)
        s = {"src": [_src_view(d["src"][i]) for i in range(d["nseg"])],
             "w": _snap(d["w"], d["w_rows"], d["w_ld"], d["w_ld"]),
             "colbias": _vec(d["colbias"], (d["nb"] - 1) * d["colbias_bstride"] + ng if d["colbias_bstride"] else ng),
             "res": _snap(d["res"], rows, d["n_valid"], d["ldr"]),
             "rowstat_in": _snap(d["rowstat_in"], rows, 2, 2, torch.int64),
             "colsum": _vec(d["colsum"], ng),
             "rowstat_out": _snap(d["rowstat_out"], rows, 2, 2, torch.int64)}
        c_out = d["col2"] if d["out2"] else d["n_valid"]
        s["spare"] = _spare(d["out"], rows, c_out, d["ldc"])
        if d["out2"]:
            s["spare2"] = _spare(d["out2"], d["n_valid"] - d["col2"], rows, d["ld2"])
        return s

    def _after_igemm(self, rec, kind, label, s):
        d = R.as_dict(rec.igemm)
        pl = R.as_dict(rec.plan)
        if kind == "igemm":
            self.tiles.add((d["nb"], d["ho"], d["wo"], pl["tw"], pl["th"], pl["tn"], pl["swap"]))
            self.branch["igemm"].add((d["nb"], d["ho"], d["wo"], pl["tw"], pl["th"], pl["tn"], pl["swap"],
                                      d["flags"] & (R.IG_SILU | R.IG_PAD0)))
        self.branch["conv"].add((kind, label.split(" ")[1]))
        cls = _kind_class(kind, d)
        atol, rtol = R.TOL[cls]
        rows, ng = R.rows_of(d), R.n_gemm(d)
        k = sum(nt * c for _, _, nt, c in R.k_segments(d))
        dtype = torch.float32 if 2.0 * rows * ng * k > R.BIG_FLOP else torch.float64
        acc = R.contraction_acc(d, s["src"], s["w"], None, dtype)
        def epi(a, dd=d, cb=s["colbias"], res=s["res"], rs=s["rowstat_in"]):
            return R.epilogue(dd, a, cb, res, rs, s["colsum"])

        ref = epi(acc)
        main, tr = R.split_out2(d, ref)
        got = _dev(d["out"], rows, main.shape[1], d["ldc"])
        units = R.tol_units(got, main, atol, rtol)
        if tr is not None:
            got2 = _dev(d["out2"], tr.shape[0], rows, d["ld2"])
            units = max(units, R.tol_units(got2, tr, atol, rtol))
        wrongs = {}

        def margin(name, wrong):
            wm, wt = R.split_out2(d, wrong)
            m = R.tol_units(wm, main, atol, rtol)
            if wt is not None:
                m = max(m, R.tol_units(wt, tr, atol, rtol))
            wrongs[name] = m

        # Part of K lost: the last split-K rank's slice, or the last K block with weights.  On images smaller than the 3x3
        # window (a 1x1 level) those blocks can hold only taps over the zero padding and change nothing; then the next rank /
        # block back is the one whose loss the check shows.
        if d["splits"] > 1:
            kps = pl["kb_per_split"]
            ranks = range(-(-pl["total_kb"] // kps) - 1, -1, -1)
            cands = [("last split-K rank lost" if i == 0 else "an earlier split-K rank lost",
                      R.k_block_mask(d, r * kps, (r + 1) * kps, acc.device)) for i, r in enumerate(ranks)]
        else:
            blocks = R.nonzero_blocks(d, s["w"])[::-1]
            cands = [("last non-zero K block dropped" if i == 0 else "an earlier non-zero K block dropped",
                      R.k_block_mask(d, b, b + 1, acc.device)) for i, b in enumerate(blocks)]
        for name, km in cands:
            margin(name, epi(R.contraction_acc(d, s["src"], s["w"], km, dtype)))
            if wrongs[name] >= 10.0:
                break
        if s["colbias"] is not None and d["colbias_bstride"] and d["nb"] > 1:
            margin("image 0's bias for every image", epi(acc, dd=dict(d, colbias_bstride=0), cb=s["colbias"][:ng]))
        if s["colsum"] is not None:
            margin("neighbouring row's LayerNorm statistics", epi(acc, rs=torch.roll(s["rowstat_in"], 1, dims=0)))
        if s["res"] is not None and d["res_scale"] != 0:
            margin("residual omitted", epi(acc, res=None))
        if s["rowstat_out"] is not None:   # the producer's fixed-point statistics of its stored fp16 rows
            delta = (_dev(d["rowstat_out"], rows, 2, 2, torch.int64) - s["rowstat_out"]).double() / R.STAT_SCALE
            want = R.rowstat_sums(got)
            x = got.double()
            bound = torch.stack([x.abs().sum(1), (x * x).sum(1)], dim=1) * 1e-4 + 1e-3
            u = ((delta - want).abs() / bound).max().item()
            self.lnstat = max(self.lnstat, u)
            assert u <= 1.0, f"{label}: LayerNorm row statistics off by {u:.3g}x their bound"
        if s["spare"] is not None:
            c_out = d["col2"] if d["out2"] else d["n_valid"]
            now = _dev(d["out"], rows - 1, d["ldc"], d["ldc"])[:, c_out:].view(torch.int16)
            assert torch.equal(now, s["spare"]), f"{label}: stray write into the spare columns [{c_out}, {d['ldc']})"
        if s.get("spare2") is not None:
            now = _dev(d["out2"], d["n_valid"] - d["col2"] - 1, d["ld2"], d["ld2"])[:, rows:].view(torch.int16)
            assert torch.equal(now, s["spare2"]), f"{label}: stray write into the V^T pad columns [{rows}, {d['ld2']})"
        self._record(cls, label, units, wrongs)

    # ---- attention ------------------------------------------------------------------------------------------------------
    def _before_attn(self, rec):
        a = R.as_dict(rec.attn)
        w = a["heads"] * a["dp"]
        return {"q": _snap(a["q"], a["nb"] * a["sq"], w, a["ldq"]), "k": _snap(a["k"], a["k_rows"], w, a["ldk"]),
                "vt": _snap(a["vt"], w, a["vt_cols"], a["ldvt"]),
                "spare": _spare(a["out"], a["nb"] * a["sq"], a["heads"] * a["d_real"], a["ldo"])}

    def _after_attn(self, rec, kind, label, s):
        a = R.as_dict(rec.attn)
        if a["k_bstride"] > 0:
            self.self_attn.add((a["nb"], a["sq"]))
        if a["dp"] == 512:
            self.branch["d512"].add(a["sq"])
        atol, rtol = R.TOL["attention"]
        ref = R.attention_ref(a, s["q"], s["k"], s["vt"])
        got = _dev(a["out"], a["nb"] * a["sq"], a["heads"] * a["d_real"], a["ldo"])
        units = R.tol_units(got, ref, atol, rtol)
        bkv = 128 if a["dp"] in (64, 128) else 64
        wrongs = {}
        if a["skv"] > bkv:
            wrongs["last KV block dropped"] = R.tol_units(R.attention_ref(a, s["q"], s["k"], s["vt"], drop_last_block=bkv), ref, atol, rtol)
        else:
            wrongs["last key dropped"] = R.tol_units(R.attention_ref(a, s["q"], s["k"], s["vt"], drop_last_block=1), ref, atol, rtol)
        # image 0's last query tile (128 rows, or the rows left after the full tiles) not written: left as zeros.  Dropping one KV
        # block moves a long sequence's output too little to show (15360 keys of the AutoencoderKL at 1024 x 960)
        tail = a["sq"] - (a["sq"] - 1) // 128 * 128
        unwritten = ref.clone()
        unwritten[a["sq"] - tail:a["sq"]] = 0
        wrongs["image 0's last query tile not written"] = R.tol_units(unwritten, ref, atol, rtol)
        if a["nb"] > 1 and a["k_bstride"] > 0:
            wrongs["image 0's K/V for every image"] = R.tol_units(R.attention_ref(a, s["q"], s["k"], s["vt"], kv_item0=True), ref, atol, rtol)
        if a["dp"] != a["d_real"]:
            wrongs["dp^-0.5 softmax scale"] = R.tol_units(R.attention_ref(a, s["q"], s["k"], s["vt"], dp_scale=True), ref, atol, rtol)
        if s["spare"] is not None:
            now = _dev(a["out"], a["nb"] * a["sq"] - 1, a["ldo"], a["ldo"])[:, a["heads"] * a["d_real"]:].view(torch.int16)
            assert torch.equal(now, s["spare"]), f"{label}: stray write into the spare output columns"
        self._record("attention", label, units, wrongs)

    # ---- GroupNorm / LayerNorm ------------------------------------------------------------------------------------------
    def _before_groupnorm(self, rec):
        g = R.as_dict(rec.groupnorm)
        rows, c = g["nb"] * g["hw"], g["ca"] + g["cb"]
        return {"xa": _snap(g["xa"], rows, g["ca"], g["lda"]), "xb": _snap(g["xb"], rows, g["cb"], g["ldb"]) if g["xb"] else None,
                "gamma": _vec(g["gamma"], c), "beta": _vec(g["beta"], c), "spare": _spare(g["y"], rows, c, g["ldy"])}

    def _after_groupnorm(self, rec, kind, label, s):
        g = R.as_dict(rec.groupnorm)
        self.branch["groupnorm"].add((g["ca"], g["cb"], g["hw"]))
        atol, rtol = R.TOL["norm"]
        rows, c = g["nb"] * g["hw"], g["ca"] + g["cb"]
        ref = R.groupnorm_ref(g, s["xa"], s["xb"], s["gamma"], s["beta"])
        got = _dev(g["y"], rows, c, g["ldy"])
        wrongs = {"neighbouring group's statistics":
                  R.tol_units(R.groupnorm_ref(g, s["xa"], s["xb"], s["gamma"], s["beta"], shift_groups=True), ref, atol, rtol)}
        if s["spare"] is not None:
            assert torch.equal(_dev(g["y"], rows - 1, g["ldy"], g["ldy"])[:, c:].view(torch.int16), s["spare"]), \
                f"{label}: stray write into the spare columns"
        self._record("norm", label, R.tol_units(got, ref, atol, rtol), wrongs)

    def _before_layernorm(self, rec):
        l = R.as_dict(rec.layernorm)
        return {"x": _snap(l["x"], l["rows"], l["c"], l["ldx"]), "gamma": _vec(l["gamma"], l["c"]),
                "beta": _vec(l["beta"], l["c"]), "spare": _spare(l["y"], l["rows"], l["c"], l["ldy"])}

    def _after_layernorm(self, rec, kind, label, s):
        l = R.as_dict(rec.layernorm)
        atol, rtol = R.TOL["norm"]
        ref = R.layernorm_ref(l, s["x"], s["gamma"], s["beta"])
        got = _dev(l["y"], l["rows"], l["c"], l["ldy"])
        # (a few rows -- one token per image of a 64 x 64 engine -- can have near-identical statistics: the affine wrong
        # reference then still shows that the check discriminates)
        wrongs = {"neighbouring row's statistics":
                  R.tol_units(R.layernorm_ref(l, s["x"], s["gamma"], s["beta"], shift_rows=True), ref, atol, rtol),
                  "neighbouring column's gamma / beta":
                  R.tol_units(R.layernorm_ref(l, s["x"], s["gamma"], s["beta"], shift_affine=True), ref, atol, rtol)}
        if s["spare"] is not None:
            assert torch.equal(_dev(l["y"], l["rows"] - 1, l["ldy"], l["ldy"])[:, l["c"]:].view(torch.int16), s["spare"]), \
                f"{label}: stray write into the spare columns"
        self._record("norm", label, R.tol_units(got, ref, atol, rtol), wrongs)

    # ---- smallconv --------------------------------------------------------------------------------------------------------
    def _before_smallconv(self, rec):
        a = R.as_dict(rec.smallconv)
        f, nb, cin = a["flags"], a["nb"], a["cin"]
        if f & (R.SC_IN_F32_NCHW | R.SC_IN_F16_NCHW):
            dt = torch.float32 if f & R.SC_IN_F32_NCHW else torch.float16
            x = _snap(a["x"], nb * cin * a["in_h"], a["in_w"], a["in_w"], dt).reshape(nb, cin, a["in_h"], a["in_w"])
        else:
            dt = torch.uint8 if f & R.SC_IN_U8 else torch.float16
            x = _snap(a["x"], nb * a["in_h"] * a["in_w"], cin, cin, dt).reshape(nb, a["in_h"], a["in_w"], cin)
        hw = a["h"] * a["w"]
        res = None
        if a["res"]:
            items = nb if a["res_bstride"] else 1
            res = torch.stack([_snap(a["res"] + 2 * n * a["res_bstride"], hw, a["cout"], a["ldr"]) for n in range(items)])
        return {"x": x, "wt": _snap(a["wt"], 9 * cin, a["cout"], a["cout"], torch.float32), "bias": _vec(a["bias"], a["cout"]),
                "in_off": _vec(a["in_off"], 3), "res": res, "spare": _spare(a["y"], nb * hw, a["cout"], a["ldy"])}

    def _after_smallconv(self, rec, kind, label, s):
        a = R.as_dict(rec.smallconv)
        if a["res"] and a["res_bstride"] == 0:
            self.branch["res_bs0"].add((label, a["nb"]))
        atol, rtol = R.TOL["smallconv"]
        rows = a["nb"] * a["h"] * a["w"]

        def ref(**kw):
            return R.smallconv_ref(a, s["x"], s["wt"], s["bias"], s["res"], s["in_off"], **kw)
        want = ref()
        got = _dev(a["y"], rows, a["cout"], a["ldy"])
        wrongs = {"3x3 taps mirrored": R.tol_units(ref(mirrored=True), want, atol, rtol)}
        if (a["in_h"] != a["h"] or a["in_w"] != a["w"]) and not (
                torch.equal(R.nearest_index(a["in_h"], a["h"]), R.nearest_index(a["in_h"], a["h"], exact_integer=True)) and
                torch.equal(R.nearest_index(a["in_w"], a["w"]), R.nearest_index(a["in_w"], a["w"], exact_integer=True))):
            wrongs["exact-integer resize rule"] = R.tol_units(ref(exact_integer=True), want, atol, rtol)
        if s["res"] is not None:
            wrongs["residual omitted"] = R.tol_units(ref(no_res=True), want, atol, rtol)
            if a["res_bstride"] and a["nb"] > 1:
                wrongs["item 0's residual for every item"] = R.tol_units(ref(res_item0=True), want, atol, rtol)
        if a["flags"] & R.SC_IN_OFFSET:
            wrongs["offset applied after the zero padding"] = R.tol_units(ref(offset_after_pad=True), want, atol, rtol)
        if s["spare"] is not None:
            now = _dev(a["y"], rows - 1, a["ldy"], a["ldy"])[:, a["cout"]:].view(torch.int16)
            assert torch.equal(now, s["spare"]), f"{label}: stray write into the spare columns [{a['cout']}, {a['ldy']})"
        self._record("smallconv", label, R.tol_units(got, want, atol, rtol), wrongs)

    # ---- upsample2x / maxpool2x2 (bit-exact) ------------------------------------------------------------------------------
    def _before_upsample2x(self, rec):
        a = R.as_dict(rec.upsample2x)
        return {"x": _snap(a["x"], a["nb"] * a["h"] * a["w"], a["c"], a["c"]).reshape(a["nb"], a["h"], a["w"], a["c"])}

    def _after_upsample2x(self, rec, kind, label, s):
        a = R.as_dict(rec.upsample2x)
        want = R.upsample2x_ref(s["x"])
        got = _dev(a["y"], a["nb"] * 4 * a["h"] * a["w"], a["c"], a["c"]).reshape(want.shape)
        ok = torch.equal(got.view(torch.int16), want.view(torch.int16))
        # (a 1x1 source has one pixel to read whichever row rule applies: the channel check still tells)
        self._record("upsample2x", label, 0.0 if ok else float("inf"),
                     {"source row (y+1)//2": _frac(R.upsample2x_ref(s["x"], shifted=True), want),
                      "channels shifted by one": _frac(R.upsample2x_ref(s["x"].roll(1, 3)), want)}, exact=True)

    def _before_maxpool2x2(self, rec):
        a = R.as_dict(rec.maxpool2x2)
        return {"x": _snap(a["x"], a["nb"] * a["h"] * a["w"], a["c"], a["c"]).reshape(a["nb"], a["h"], a["w"], a["c"])}

    def _after_maxpool2x2(self, rec, kind, label, s):
        a = R.as_dict(rec.maxpool2x2)
        self.branch["maxpool2x2"].add((a["h"], a["w"], a["c"]))
        want = R.maxpool2x2_ref(s["x"])
        got = _dev(a["y"], a["nb"] * (a["h"] // 2) * (a["w"] // 2), a["c"], a["c"]).reshape(want.shape)
        ok = torch.equal(got.view(torch.int16), want.view(torch.int16))
        self._record("maxpool2x2", label, 0.0 if ok else float("inf"),
                     {"average pooling": _frac(R.maxpool2x2_ref(s["x"], average=True), want),
                      "window shifted by one": _frac(R.maxpool2x2_ref(s["x"], shifted=True), want)}, exact=True)

    # ---- HED ----------------------------------------------------------------------------------------------------------------
    def _before_hed_project(self, rec):
        a = R.as_dict(rec.hed_project)
        return {"x": _snap(a["x"], a["npix"], a["c"], a["ldx"]), "w": _vec(a["w"], a["c"]), "bias": _vec(a["bias"], 1)}

    def _after_hed_project(self, rec, kind, label, s):
        a = R.as_dict(rec.hed_project)
        atol, rtol = R.TOL["hed_project"]
        want = R.hed_project_ref(s["x"], s["w"], s["bias"])
        got = _dev(a["out"], 1, a["npix"], a["npix"], torch.float32).flatten()
        wrongs = {"bias omitted": R.tol_units(R.hed_project_ref(s["x"], s["w"], s["bias"], no_bias=True), want, atol, rtol),
                  "channel pairs swapped": R.tol_units(R.hed_project_ref(s["x"], s["w"], s["bias"], swap_pairs=True), want, atol, rtol)}
        self._record("hed_project", label, R.tol_units(got, want, atol, rtol), wrongs)

    def _before_hed_fuse(self, rec):
        a = R.as_dict(rec.hed_fuse)
        return {"maps": [_snap(a["maps"][k], a["hs"][k], a["ws"][k], a["ws"][k], torch.float32) for k in range(a["levels"])]}

    def _after_hed_fuse(self, rec, kind, label, s):
        a = R.as_dict(rec.hed_fuse)
        h, w = a["h"], a["w"]
        self.branch["hed_fuse"].add((h, w))
        got = _dev(a["out"], h * w, 3, 3, torch.uint8)
        assert torch.equal(got[:, 1], got[:, 0]) and torch.equal(got[:, 2], got[:, 0]), f"{label}: the 3 channels differ"
        u = got[:, 0].reshape(h, w)
        if a["edge_f16"]:
            assert torch.equal(_dev(a["edge_f16"], h * w, 1, 1).reshape(h, w), u.half()), f"{label}: edge_f16 != the u8 value"
        nbad, near = R.hed_fuse_mismatch(u, s["maps"], h, w)
        assert near, f"{label}: a pixel off by more than 1, or away from an integer boundary"
        want = R.hed_fuse_ref(s["maps"], h, w)
        self._record("hed_fuse", label, nbad / (1e-3 * h * w),
                     {"align_corners=True": _frac(R.hed_fuse_ref(s["maps"], h, w, align_corners=True), want),
                      "rounding instead of truncation": _frac(R.hed_fuse_ref(s["maps"], h, w, rounding=True), want)}, exact=True)

    # ---- scheduler step (rewrites the stream-batch buffer in place) ----------------------------------------------------------
    def _before_lcm_step(self, rec):
        a = R.as_dict(rec.lcm_step)
        n = a["T"] * a["hw"]
        return {"x": _snap(a["x"], n, 4, 4), "eps": _snap(a["eps"], n, 4, 4), "noise": _snap(a["noise"], n, 4, 4),
                "coef": _vec(a["coef"], 4 * a["T"])}

    def _after_lcm_step(self, rec, kind, label, s):
        a = R.as_dict(rec.lcm_step)
        T, hw = a["T"], a["hw"]
        self.stream_batch.add(T)
        atol, rtol = R.TOL["lcm_step"]
        noise = s["noise"] if s["noise"] is not None else torch.zeros_like(s["x"])
        args = (a, s["x"].reshape(T, hw, 4), s["eps"].reshape(T, hw, 4), noise.reshape(T, hw, 4), s["coef"])
        out, x = R.lcm_step_ref(*args)
        got_out = _dev(a["out_latent"], hw, 4, 4)
        got_x = _dev(a["x"], T * hw, 4, 4).reshape(T, hw, 4)

        def units(go, gx):   # distance of (out_latent, x) from the reference, in tolerance units
            u = R.tol_units(go, out, atol, rtol)
            return max(u, R.tol_units(gx[1:], x[1:], atol, rtol)) if T > 1 else u
        assert torch.equal(got_x[0].view(torch.int16), s["x"][:hw].view(torch.int16)), f"{label}: slot 0 of x changed"
        assert torch.equal(_dev(a["eps"], T * hw, 4, 4), s["eps"]), f"{label}: eps changed"
        if s["noise"] is not None:
            assert torch.equal(_dev(a["noise"], T * hw, 4, 4), s["noise"]), f"{label}: noise changed"
        wrongs = {"c_skip / c_out swapped": units(*R.lcm_step_ref(*args, swap_cskip_cout=True))}
        if T > 1:
            wrongs["slot i re-noised from its own x0"] = units(*R.lcm_step_ref(*args, own_x0=True))
        self._record("lcm_step", label, units(got_out, got_x), wrongs)

    # ---- post_u8 (bit-exact) ------------------------------------------------------------------------------------------------
    def _before_post_u8(self, rec):
        a = R.as_dict(rec.post_u8)
        return {"y": _snap(a["y"], a["nb"] * a["h"] * a["w"], 3, a["ldy"])}

    def _after_post_u8(self, rec, kind, label, s):
        a = R.as_dict(rec.post_u8)
        want = R.post_u8_ref(a, s["y"])
        got = _dev(a["out"], a["nb"] * 3 * a["h"], a["w"], a["w"], torch.uint8).reshape(want.shape)
        self._record("post_u8", label, 0.0 if torch.equal(got, want) else float("inf"),
                     {"rounding instead of truncation": _frac(R.post_u8_ref(a, s["y"], rounding=True), want),
                      "BGR channel order": _frac(R.post_u8_ref(a, s["y"], bgr=True), want)}, exact=True)

    # ---- prepare-time: time embedding ---------------------------------------------------------------------------------------
    def _before_small_linear(self, rec):
        a = R.as_dict(rec.small_linear)
        return {"x": _snap(a["in"], a["nb"], a["k"], a["in_ld"], torch.float32), "w": _snap(a["w"], a["n"], a["k"], a["k"]),
                "bias": _vec(a["bias"], a["n"])}

    def _after_small_linear(self, rec, kind, label, s):
        a = R.as_dict(rec.small_linear)
        atol, rtol = R.TOL["small_linear"]

        def ref(**kw):
            return R.small_linear_ref(a, s["x"], s["w"], s["bias"], **kw)
        want = ref()
        got = _dev(a["out"], a["nb"], a["n"], a["out_ld"], torch.float32)
        wrongs = {}
        if a["silu_in"]:
            wrongs["SiLU omitted"] = R.tol_units(ref(no_silu=True), want, atol, rtol)
        if s["bias"] is not None:
            wrongs["bias omitted"] = R.tol_units(ref(no_bias=True), want, atol, rtol)
        if a["nb"] > 1:
            wrongs["slot 0's input for every slot"] = R.tol_units(ref(slot0=True), want, atol, rtol)
        self._record("small_linear", label, R.tol_units(got, want, atol, rtol), wrongs)

    def _before_timestep_embedding(self, rec):
        a = R.as_dict(rec.timestep_embedding)
        return {"t": _vec(a["t"], a["nb"])}

    def _after_timestep_embedding(self, rec, kind, label, s):
        a = R.as_dict(rec.timestep_embedding)
        want = R.timestep_embedding_ref(s["t"], a["dim"])
        got = _dev(a["out"], a["nb"], a["dim"], a["dim"], torch.float32).double()

        def units(x):
            return (x - want).abs().max().item() / R.TEMB_ATOL
        self._record("timestep_embedding", label, units(got),
                     {"[sin | cos] order": units(R.timestep_embedding_ref(s["t"], a["dim"], sin_first=True)),
                      "exponent over half - 1": units(R.timestep_embedding_ref(s["t"], a["dim"], half_minus_one=True))})

    def table(self, name):
        lines = [f"launch audit {name}: {self.calls} launches, {sum(self.other.values())} other",
                 f"  {'class':16s} {'launches':>8s} {'checked':>8s} {'worst/tol':>9s}  wrong references applied (worst launch)"]
        for cls in sorted(self.launches):
            wr = ", ".join(f"{k}: {v}" for k, v in sorted(self.wrong[cls].items()))
            lines.append(f"  {cls:16s} {self.launches[cls]:8d} {self.checked[cls]:8d} {self.worst[cls]:9.3f}  {wr}  "
                         f"({self.worst_label.get(cls, '')})")
        lines.append("  other launches by label: " + ", ".join(f"{k}: {v}" for k, v in sorted(self.other.items())))
        lines.append(f"  LayerNorm statistics producers: worst {self.lnstat:.3g}x their bound")
        return "\n".join(lines)


def _engine(turbo, tl, hw, full=False, concurrency=1, cn=False, hed=False, kl=False):
    from ai_rtc_agent_b200.host import arch as A
    from ai_rtc_agent_b200.host.stream import StreamDiffusion
    from oracle import controlnet as ocn
    from oracle import unet as ounet
    from oracle import weights as ow
    height, width = (hw, hw) if isinstance(hw, int) else hw
    if full:
        cfg, arch = (ounet.SD_TURBO, A.SD_TURBO) if turbo else (ounet.SD15, A.SD15)
        varch = A.AUTOENCODER_KL
    else:
        cfg, arch, varch = ounet.tiny_config(turbo), (A.TINY_TURBO if turbo else A.TINY_SD15), A.TINY_AUTOENCODER_KL
    usd = ow.make_unet_weights(cfg)
    vsd = A.synthetic_autoencoder_kl(varch) if kl else ow.make_taesd_weights()
    emb = ow.make_prompt_embeds(cfg.cross_attention_dim)
    cn16 = ocn.make_weights(cfg) if cn else None
    hed16 = {k: v.half().float() for k, v in A.synthetic_hed().items()} if hed else None
    sd = StreamDiffusion(arch, usd, vsd, tl, lambda p: emb, width=width, height=height, device="cuda", use_tiny_vae=not kl,
                         controlnet_sd=cn16, hed_sd=hed16)
    if concurrency > 1:
        sd.set_concurrency(concurrency)
    sd.prepare("p", guidance_scale=0.0)
    lane = sd.add_lane()
    # a lane defaults to the launch policy of >= 2 frames in flight (other split-K factors, other summation order): give it
    # the audited engine's policy, so that the two compute bit-identical frames
    lane.set_concurrency(concurrency)
    lane._prepare_like(sd)
    keys = list(usd) + (list(cn16) if cn else [])   # the UNet's and the ControlNet's parameters
    return sd, lane, keys


_TINY = [
    pytest.param(dict(turbo=True, tl=[32], hw=128), id="tiny-turbo-T1-128"),
    pytest.param(dict(turbo=False, tl=_T4, hw=(128, 192)), id="tiny-sd15-T4-128x192"),
    pytest.param(dict(turbo=False, tl=_T4, hw=192), id="tiny-sd15-T4-192"),             # unfolded transformer program: 36 / 9 tokens
    pytest.param(dict(turbo=True, tl=[32], hw=192, cn=True, hed=True), id="tiny-turbo-T1-192-cn-hed"),
    pytest.param(dict(turbo=False, tl=_T4, hw=128, kl=True), id="tiny-sd15-T4-128-kl"),
    # a camera-sized frame: the heads resize 300x400 -> 128x192 (400 -> 192: torch's rule and the integer rule differ), and
    # the ControlNet head writes 16 channels into a 64-wide buffer
    pytest.param(dict(turbo=True, tl=[32], hw=(128, 192), cn=True, frame=(300, 400)), id="tiny-turbo-T1-128x192-cn-300x400"),
]
_FULL = [
    pytest.param(dict(turbo=True, tl=[32], hw=512, concurrency=1), id="turbo-T1-512-c1"),
    pytest.param(dict(turbo=True, tl=[32], hw=512, concurrency=8), id="turbo-T1-512-c8"),
    pytest.param(dict(turbo=False, tl=_T4, hw=512, concurrency=1), id="sd15-T4-512-c1"),
    pytest.param(dict(turbo=False, tl=_T4, hw=512, concurrency=4), id="sd15-T4-512-c4"),
    pytest.param(dict(turbo=False, tl=_T4, hw=448, concurrency=1), id="sd15-T4-448-c1"),   # unfolded program at 14x14 (level 2)
    pytest.param(dict(turbo=True, tl=[32], hw=512, cn=True, hed=True), id="turbo-T1-512-cn-hed"),
    pytest.param(dict(turbo=True, tl=[32], hw=512, kl=True), id="turbo-T1-512-kl"),
    # 720 -> 448 is a pair where torch's rule and the integer rule differ; the 448x768 head runs 64-channel groups and the
    # grid-stride loop
    pytest.param(dict(turbo=True, tl=[32], hw=(448, 768), frame=(720, 1280)), id="turbo-T1-448x768-720x1280"),
    # stream batch 3 at the 8x8 level: a phantom image in the last M tile of the 1280-channel contractions, with split-K
    pytest.param(dict(turbo=False, tl=[18, 30, 45], hw=512, concurrency=1), id="sd15-T3-512-c1"),
    pytest.param(dict(turbo=False, tl=_T4, hw=768, concurrency=1), id="sd15-T4-768-c1"),   # the golden configuration
    # 16384-token self-attention, the fused / statistics + apply GroupNorms of the up path, CTA pairs
    pytest.param(dict(turbo=True, tl=[32], hw=1024, concurrency=8), id="turbo-T1-1024-c8"),
]


def _release_device_memory():
    """Engines allocate with cudaMalloc, outside torch's caching allocator: hand torch's cached blocks (earlier tests' references
    and snapshots) back to the driver, and collect engines that only a reference cycle keeps alive (a parent and its lanes
    refer to each other), so that each configuration starts with the HBM that it alone needs."""
    gc.collect()
    torch.cuda.empty_cache()


def _audit(cuda, name, cfg, full):
    from oracle import weights as ow
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    sd = lane = None
    _release_device_memory()
    free0 = torch.cuda.mem_get_info()[0]
    cfg = dict(cfg)
    frame_hw = cfg.pop("frame", None)
    try:
        t0 = time.time()
        sd, lane, keys = _engine(full=full, **cfg)
        fh, fw = frame_hw or (sd.height, sd.width)
        nframes = 2 if len(cfg["tl"]) > 1 else 1      # T = 4: the second frame runs on a non-zero latent buffer
        frames = [ow.make_frame(fh, fw, seed=300 + i).cuda() for i in range(nframes)]
        for f in frames[:-1]:
            sd.step_u8(f)
            lane.step_u8(f)
        # the refresh recomputes sd's time biases and prompt K / V^T: the bit-identity with the lane below also shows that
        # it is deterministic
        ref_aud = Auditor()
        sd.audit_refresh(ref_aud)
        aud = Auditor()
        got = sd.audit_step(frames[-1], aud).clone()
        want = lane.step_u8(frames[-1])
        torch.cuda.synchronize()
        peak = free0 - min(a.min_free for a in (ref_aud, aud) if a.min_free is not None)
        print("\n" + ref_aud.table(name + " refresh") + "\n" + aud.table(name) + f"\n  wall time {time.time() - t0:.1f} s, "
              f"free HBM at the start {free0 / 2**30:.1f} GiB, peak in use during the audit {peak / 2**30:.1f} GiB")
        for a in (ref_aud, aud):
            assert not a.other, f"launches without a record: {dict(a.other)}"
            for cls in a.launches:
                assert a.checked[cls] == a.launches[cls], cls
            assert a.calls == sum(a.checked.values())
        # the frame: every class it must have, the scheduler step and the tail exactly once, HED only with HED
        assert aud.calls == sd.launches_per_step, (aud.calls, sd.launches_per_step)
        assert {"contraction", "attention", "norm", "smallconv", "upsample2x", "lcm_step", "post_u8"} <= set(aud.checked), \
            dict(aud.checked)
        assert aud.checked["lcm_step"] == 1 and aud.checked["post_u8"] == 1, dict(aud.checked)
        hed = {k: aud.checked[k] for k in _HED if aud.checked[k]}
        assert hed == ({"maxpool2x2": 4, "hed_project": 5, "hed_fuse": 1} if cfg.get("hed") else {}), hed
        # the refresh, tied to the model: one time-bias projection per resnet with a time embedding, one time MLP (two
        # linears) per model, and the K and V^T projections of every cross attention
        n_temb = sum(k.endswith("time_emb_proj.weight") for k in keys)
        n_attn2 = sum(k.endswith("attn2.to_k.weight") for k in keys)
        nets = 2 if cfg.get("cn") else 1
        assert ref_aud.checked["timestep_embedding"] == 1, dict(ref_aud.checked)
        assert ref_aud.labels["small_linear", "temb"] == n_temb > 0, (dict(ref_aud.labels), n_temb)
        assert ref_aud.checked["small_linear"] == n_temb + 2 * nets, (dict(ref_aud.checked), n_temb)
        assert ref_aud.checked["contraction"] == 2 * n_attn2 > 0, (dict(ref_aud.checked), n_attn2)
        assert set(ref_aud.checked) == {"timestep_embedding", "small_linear", "contraction"}, dict(ref_aud.checked)
        assert torch.equal(got, want), "the audited frame differs from a graph step of an identical lane"
        return aud
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
        if sd is not None:
            sd.lanes.clear()   # break the parent <-> lane cycle: both engines are destroyed here, not at some later collection
        sd = lane = None
        _release_device_memory()


@pytest.mark.parametrize("cfg", _TINY)
def test_frame_and_refresh_launch_audit_tiny(cuda, request, cfg):
    _audit(cuda, request.node.callspec.id, cfg, full=False)


@pytest.mark.parametrize("cfg", _FULL)
def test_frame_and_refresh_launch_audit_full_size(cuda, request, cfg):
    _audit(cuda, request.node.callspec.id, cfg, full=True)
