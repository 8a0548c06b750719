"""Host-side launch planning (tile / split-K policy of the frame program, GroupNorm launch shapes) evaluated WITHOUT a GPU
through the C ABI's dry-run entry points: invariants over every contraction shape of the two UNets and TAESD plus a random
sweep, and the policy decisions taken from cold-weight sweeps (tools/bench_op.py) pinned as regression cases."""
import ctypes as C
import random

import pytest

from ai_rtc_agent_b200.host import capi

SMEM_MAX = 227 * 1024
SMS = 132   # H100 SXM streaming multiprocessors
RING_KB = 200   # operand ring of a launch whose CTAs each have an SM to themselves (igemm: one resident CTA per SM)


def _full_ring_stages(info):
    """Stages a plan gets when nothing cuts its ring to share an SM: as many as the 200 KB budget holds, within [2, 8] and the
    K-blocks of its slice (split-K staging may grow it further)."""
    stage = 128 * 128 + info.bn * 128
    return max(2, min(8, RING_KB * 1024 // stage, max(2, info.kb_per_split)))


def _desc(nb, h, w, srcs, cout, stride=1, bn=0, splits=1, swap=0, geglu=False, res=False, flags=0):
    """srcs: [(channels, ntap)], output h/stride x w/stride x cout; flags: further epilogue / kernel-variant flags (IG_SILU,
    IG_PAD0), which restrict the planner's choices as they do in the engine"""
    d = capi.IgemmDesc()
    d.nseg = len(srcs)
    k = 0
    for i, (c, ntap) in enumerate(srcs):
        d.src[i].ptr = 0x100000 * (i + 1)
        d.src[i].n, d.src[i].h, d.src[i].w, d.src[i].c, d.src[i].ld = nb, h, w, c, c
        d.ntap[i] = ntap
        k += c * ntap
    d.w, d.w_rows, d.w_ld = 0x4000000, cout * (2 if geglu else 1), k
    d.stride = stride
    d.nb, d.ho, d.wo = nb, h // stride, w // stride
    d.bn, d.splits, d.swap = bn, splits, swap
    d.out, d.ldc = 0x8000000, cout
    d.colbias, d.colbias_bstride = 0xA000000, cout * (2 if geglu else 1)
    if res:
        d.res, d.ldr = 0xC000000, cout
    d.acc_scale = d.res_scale = 1.0
    d.flags = (capi.IG_GEGLU if geglu else 0) | flags
    d.n_valid = cout
    return d, k // 64


def _plan(d, autotile=1, allow_swap=0):
    info = capi.IgemmPlanInfo()
    rc = capi.lib().b2sd_igemm_plan_dry(C.byref(d), autotile, allow_swap, C.byref(info))
    assert rc == 0, capi.lib().b2sd_last_error()
    return info


def _check(info, d, total_kb, geglu=False, pairs_ok=False):
    n_gemm = d.n_valid * (2 if geglu else 1)
    rows = d.nb * d.ho * d.wo
    assert info.mode in ((0, 1) if pairs_ok else (0,)) and info.rows_total == rows and info.total_kb == total_kb
    if info.mode == 1:   # CTA pairs: x = pairs of neighbouring M tiles, cluster (2, 1, splits) within the portable limit of 8
        assert not info.swap and info.bn % 32 == 0 and info.splits in (1, 2, 4) and info.grid_x % 2 == 0 and info.m_tiles >= 2
    assert info.splits in (1, 2, 4, 8) and info.grid_z == info.splits
    assert info.kb_per_split * info.splits >= total_kb > info.kb_per_split * (info.splits - 1), "empty or missing K slice"
    assert 2 <= info.num_stages <= 8
    assert info.smem_bytes <= SMEM_MAX
    assert info.tmem_cols in (32, 64, 128, 256, 512) and info.tmem_cols >= info.bn * info.acc_bufs
    if info.splits > 1:
        assert info.acc_bufs == 1
        assert info.bn * 128 * 4 <= info.smem_bytes - 1536, "split-K staging tile does not fit the operand ring"
    if info.swap:
        assert info.bn in (64, 128, 256) and info.grid_y * 128 >= d.n_valid and info.grid_x * info.bn >= rows
    else:
        assert info.bn % 16 == 0 and 16 <= info.bn <= 256 and info.grid_y * info.bn >= n_gemm
        assert info.m_tiles * 128 >= rows
        if info.acc_bufs == 2:   # persistent over M tiles
            # one resident wave (at least one CTA per N tile, a pair of them for CTA pairs)
            assert info.grid_x * info.grid_y <= max(SMS, info.grid_y * (2 if info.mode == 1 else 1)) and SMS < info.m_tiles * info.grid_y and info.grid_x <= info.m_tiles
        else:
            assert info.grid_x == (info.m_tiles + 1) // 2 * 2 if info.mode == 1 else info.grid_x == info.m_tiles


def _unet_shapes(chs, nb, lh=64, lw=64):
    """(nb, (h, w), srcs, cout, stride, geglu, allow_swap) of every contraction family of a UNet with block channels `chs` on an
    lh x lw latent"""
    out = []
    res = [(lh >> k, lw >> k) for k in range(4)]
    for lvl, (c, r) in enumerate(zip(chs, res)):
        cin_prev = chs[max(lvl - 1, 0)]
        out += [(r, [(cin_prev, 9)], c, 1, False, True), (r, [(c, 9)], c, 1, False, True),          # resnet conv1 / conv2
                (r, [(c, 9), (cin_prev, 1)], c, 1, False, True)]                                          # conv2 + 1x1 shortcut
        for skip in {c, cin_prev, chs[min(lvl + 1, 3)]}:                                                # up-block concat inputs
            out.append((r, [(c, 9), (skip, 9)], c, 1, False, True))
            out.append((r, [(c, 9), (c, 1), (skip, 1)], c, 1, False, True))
        if lvl < 3:
            out += [(r, [(c, 1)], c, 1, False, True), (r, [(c, 1)], 2 * c, 1, False, True),               # proj / q,k
                    (r, [(c, 1)], 4 * c, 1, True, False), (r, [(4 * c, 1)], c, 1, False, True),           # GEGLU, FF out
                    (r, [(c, 9)], c, 2, False, True)]                                                   # downsampler
    return [(nb,) + s for s in out]


def _latent_cases(cases):
    """(nb, lh, lw) parameters; square latents keep their "nb-latent" ids"""
    return [pytest.param(nb, lh, lw, id=f"{nb}-{lh}" if lh == lw else f"{nb}-{lh}x{lw}") for nb, lh, lw in cases]


# non-square engines: 384x512 (SD-Turbo 6x8 level on the swapped path), 448x768, 768x448 (Wo = 7 at the 12x7 level) and the
# 128x192 tiny size (2x3 level, several images in one M tile)
_NONSQUARE = [(1, 48, 64), (1, 56, 96), (4, 96, 56), (4, 16, 24)]


@pytest.mark.parametrize("nb,lh,lw", _latent_cases([(1, 64, 64), (4, 64, 64), (4, 96, 96), (1, 32, 32)] + _NONSQUARE))
def test_autotile_invariants_over_the_frame_program(nb, lh, lw):
    """BASELINE.json configs: 512x512 at stream batch 1 / 4, 768x768 at batch 4, 256x256 at batch 1; and non-square engines"""
    shapes = _unet_shapes([320, 640, 1280, 1280], nb, lh, lw)
    shapes += [(1, (lh * 8 >> k, lw * 8 >> k), [(64, 9)], 64, 1, False, False) for k in range(4)]   # TAESD body (one frame)
    shapes += [(1, (lh * 8 >> k, lw * 8 >> k), [(64, 9)], 64, 2, False, False) for k in range(3)]
    for (b, (rh, rw), srcs, cout, stride, geglu, allow_swap) in shapes:
        d, kb = _desc(b, rh, rw, srcs, cout, stride=stride, geglu=geglu)
        info = _plan(d, 1, int(allow_swap))
        _check(info, d, kb, geglu)
        ctas = info.grid_x * info.grid_y * info.grid_z
        if not info.swap:   # one CTA per SM: no launch cuts its operand ring to share an SM, however many CTAs it has
            assert info.num_stages >= _full_ring_stages(info), \
                f"{ctas} CTAs: ring of {info.num_stages} stages ({srcs}->{cout} @{rh}x{rw})"


@pytest.mark.parametrize("nb,lh,lw", _latent_cases([(1, 64, 64), (4, 64, 64), (4, 96, 96)] + _NONSQUARE))
def test_throughput_policy_invariants(nb, lh, lw):
    """autotile = 2: what the engine plans with >= 4 frames in flight (CTA pairs without split-K, full operand rings)"""
    shapes = _unet_shapes([320, 640, 1280, 1280], nb, lh, lw)
    paired = 0
    for (b, (rh, rw), srcs, cout, stride, geglu, allow_swap) in shapes:
        d, kb = _desc(b, rh, rw, srcs, cout, stride=stride, geglu=geglu)
        info = _plan(d, 2, int(allow_swap))
        _check(info, d, kb, geglu, pairs_ok=True)
        single = _plan(d, 1, int(allow_swap))
        if info.mode == 1:
            paired += 1
            assert info.splits == 1 and info.num_stages >= _full_ring_stages(info), "CTAs of different frames never share an SM"
            assert info.num_stages >= 2 and (info.bn != 160 or info.num_stages >= 3 or info.total_kb < 3)
        else:
            assert info.swap or info.m_tiles < 2 or info.bn % 32 != 0, "an eligible contraction was left on single CTAs"
        del single
    assert paired >= len(shapes) // 2


def test_throughput_policy_is_pinned():
    """Throughput launch policy (>= 4 frames in flight); a change here needs a new measurement."""
    def pol(r, srcs, cout, allow_swap=1, **kw):
        d, _ = _desc(1, r, r, srcs, cout, **kw)
        i = _plan(d, 2, allow_swap)
        return (i.mode, i.bn, i.splits, i.swap, i.grid_x, i.grid_y, i.num_stages)
    assert pol(64, [(320, 9)], 320) == (1, 160, 1, 0, 32, 2, 5)          # 36 KB stages (whole multicast weight tile): five fit 200 KB
    assert pol(32, [(1280, 9)], 640)[:3] == (1, 160, 1)
    assert pol(16, [(1280, 9)], 1280)[:6] == (1, 64, 1, 0, 2, 20)        # two M tiles = one pair per N tile, 180 K-blocks each
    assert pol(8, [(1280, 9)], 1280)[:4] == (0, 64, 4, 1)                # one M tile: stays swapped, split-K capped at 4
    assert pol(64, [(320, 1)], 1280, allow_swap=0, geglu=True)[:3] == (1, 256, 1)   # persistent pairs: 128 value + 128 gate rows per tile
    explicit, _ = _desc(1, 64, 64, [(320, 9)], 320, bn=160, splits=4)
    explicit.flags |= capi.IG_PAIR
    i = _plan(explicit, 0)
    assert (i.mode, i.grid_x, i.grid_y, i.grid_z) == (1, 32, 2, 4)
    odd, _ = _desc(1, 24, 24, [(128, 9)], 64, bn=64)                     # 5 M tiles -> 3 pairs, the last one half masked
    odd.flags |= capi.IG_PAIR
    assert _plan(odd, 0).grid_x == 6
    bad, _ = _desc(1, 64, 64, [(320, 9)], 320, bn=80)
    bad.flags |= capi.IG_PAIR
    info = capi.IgemmPlanInfo()
    assert capi.lib().b2sd_igemm_plan_dry(C.byref(bad), 0, 0, C.byref(info)) != 0, "pairs need an N tile that is a multiple of 32"


def test_autotile_random_sweep():
    rng = random.Random(1234)
    for _ in range(400):
        nb = rng.choice([1, 1, 2, 4])
        r = rng.choice([8, 16, 24, 32, 64, 96])
        nseg = rng.choice([1, 1, 2, 3])
        srcs = [(64 * rng.randint(1, 40), rng.choice([1, 9])) for _ in range(nseg)]
        cout = rng.choice([64, 128, 192, 320, 640, 1280, 2560, 96, 48])
        geglu = rng.random() < 0.15 and cout % 64 == 0
        if any(t == 9 for _, t in srcs) and geglu:
            geglu = False
        d, kb = _desc(nb, r, r, srcs, cout, geglu=geglu)
        info = _plan(d, 1, int(rng.random() < 0.5 and not geglu))
        _check(info, d, kb, geglu)


@pytest.mark.parametrize("bn,splits,swap", [(64, 1, 0), (64, 4, 0), (160, 4, 0), (256, 8, 0), (128, 2, 0), (256, 8, 1), (64, 8, 1), (128, 1, 1)])
def test_explicit_plans(bn, splits, swap):
    d, kb = _desc(1, 16, 16, [(1280, 9)], 1280, bn=bn, splits=splits, swap=swap, res=True)
    info = _plan(d, 0)
    _check(info, d, kb)
    assert (info.bn, info.splits, info.swap) == (bn, splits, swap)


def test_measured_policy_is_pinned():
    """Decisions taken from the cold-weight sweep (tools/bench_op.py); a change here needs a new measurement."""
    def pol(r, srcs, cout, allow_swap=1, **kw):
        d, _ = _desc(1, r, r, srcs, cout, **kw)
        i = _plan(d, 1, allow_swap)
        return (i.bn, i.splits, i.swap, i.acc_bufs)
    assert pol(64, [(320, 9)], 320) == (160, 4, 0, 1)
    assert pol(64, [(640, 9), (320, 9)], 320)[:2] == (160, 4)
    assert pol(32, [(640, 9)], 640) == (160, 4, 0, 1)
    assert pol(16, [(1280, 9)], 1280) == (256, 8, 0, 1)
    assert pol(8, [(1280, 9)], 1280) == (64, 8, 1, 1)                # swapped orientation at the 8x8 level
    assert pol(8, [(1280, 9)], 1280, allow_swap=0)[2] == 0
    assert pol(64, [(320, 1)], 320) == (64, 1, 0, 2)                  # 160 tiles: more than one wave of 132, persistent
    assert pol(32, [(640, 1)], 640) == (64, 1, 0, 1)                  # 80 CTAs, no split for 10 K-blocks
    assert pol(16, [(1280, 1)], 1280) == (64, 4, 0, 1)
    bn, splits, swap, acc = pol(512, [(64, 9)], 64, allow_swap=0)     # TAESD 512x512: persistent over M tiles
    assert (bn, splits, swap, acc) == (64, 1, 0, 2)
    d, _ = _desc(1, 32, 32, [(640, 9)], 640)
    assert _plan(d, 1, 1).num_stages >= 5, "<= one CTA per SM: the launch takes the 200 KB ring"


def test_bad_descriptors_are_rejected():
    d, _ = _desc(1, 16, 16, [(100, 1)], 64)          # channels not a multiple of 64
    info = capi.IgemmPlanInfo()
    assert capi.lib().b2sd_igemm_plan_dry(C.byref(d), 0, 0, C.byref(info)) != 0
    assert b"multiple of 64" in capi.lib().b2sd_last_error()
    d, _ = _desc(1, 16, 16, [(128, 1)], 100, swap=1)   # swapped epilogue needs n % 8 == 0
    assert capi.lib().b2sd_igemm_plan_dry(C.byref(d), 0, 0, C.byref(info)) != 0


def test_groupnorm_last_path_is_per_thread():
    """b2sd_groupnorm_last_path reports the launch made on the calling thread: -1 on a thread that has launched none."""
    import threading
    got = []
    t = threading.Thread(target=lambda: got.append(capi.lib().b2sd_groupnorm_last_path()))
    t.start()
    t.join()
    assert got == [-1]


@pytest.mark.parametrize("ca,cb,hw,expect", [(320, 0, 4096, 4), (640, 320, 4096, 8), (640, 0, 1024, 2), (1280, 640, 1024, 4),
                                             (1280, 0, 256, 1), (1280, 1280, 64, 1), (640, 320, 96 * 96, 0), (100, 0, 64, None)])
def test_groupnorm_launch_shape(ca, cb, hw, expect):
    cl, th, ppc = C.c_int(), C.c_int(), C.c_int()
    assert capi.lib().b2sd_groupnorm_plan_dry(ca, cb, 32, hw, C.byref(cl), C.byref(th), C.byref(ppc)) == 0
    if expect is not None:
        assert cl.value == expect
    if cl.value:
        cpg = (ca + cb) // 32
        assert cl.value in (1, 2, 4, 8) and th.value == 240 and th.value % (cpg // 2) == 0
        assert ppc.value * cl.value >= hw > ppc.value * (cl.value - 1), "pixel ranges of the cluster CTAs must tile the image"
        pstep = th.value // (cpg // 2)
        assert -(-ppc.value // pstep) <= 32, "a thread keeps at most 32 half2 words in registers"
