"""The master-weight optimizer steps where kernels go wrong: IEEE edge values in gradients, masters
and optimizer state, the half-precision write-back at its overflow thresholds and rounding ties, and
hyperparameters at their boundaries.

Every step kernel (SGD, Adam / AdamW, LAMB; plain, clipped and unscaled) must give the bits of the
stock restatements the other suites use (master_weight.Reference) in parameters, masters,
momentum_buffer, exp_avg, exp_avg_sq, max_exp_avg_sq, step and grad_norm, raw bits compared, so NaN
sign and payload and the sign of zero count.

Values come from three catalogues (gradients per half dtype, fp32 masters, optimizer state), each
tiled with an odd cycle length over a randn background, so every value lands in every lane of the 8-
and 4-wide groups.  The first step takes catalogue gradients on fresh state (SGD's `m = g`); then
catalogue masters (parameters set to half(master)) and state are written into both sides, and three
more steps carry NaN and inf through the moments.  Parameters are views at offsets chosen
so that the SGD / Adam kernels take the scalar head, 16-byte vectors with the gradient aligned and
unaligned, the scalar tail, all-scalar segments and chunk boundaries, and the LAMB kernels both
_foreach_norm accumulator mappings and both apply paths.  Before anything is compared, the kernels'
path choice is restated from the real data pointers and every catalogue entry must reach every path.
"""
import numpy as np
import pytest

import harness
from master_weight import INIT_SCALE, INTERVAL, WD, RefLAMB, Reference, bits, new_loss_scale, \
    same_bits, sched, scaling_matches, state_mismatches, stock

pytestmark = pytest.mark.gpu

CHUNK = 4096          # TOK_SGD_CHUNK: SGD / Adam work items
NORM_CHUNK = 65536    # TOK_NORM_CHUNK: LAMB work items
STEPS = 4             # step 0 on fresh state, then the catalogue state is written, then 3 more

# ---- the catalogues ------------------------------------------------------------------------------
# Gradients as raw half bits.  bf16 also has values whose fp32 square overflows (|g| >= 2^64), is an
# fp32 subnormal (2^-70) or rounds to zero (2^-80).
GRAD_CATALOGUE = {
    "bf16": (("pos_zero", 0x0000), ("neg_zero", 0x8000), ("min_subnormal", 0x0001),
             ("max_subnormal", 0x007F), ("neg_subnormal", 0x8003), ("min_normal", 0x0080),
             ("max_finite", 0x7F7F), ("neg_max_finite", 0xFF7F), ("pos_inf", 0x7F80),
             ("neg_inf", 0xFF80), ("qnan", 0x7FC0), ("nan_payload", 0x7FE5), ("neg_nan", 0xFFC0),
             ("snan", 0x7F81), ("square_overflows", 0x5F80), ("neg_square_overflows", 0xDFC0),
             ("square_subnormal", 0x1C80), ("neg_square_subnormal", 0x9CC0),
             ("square_rounds_to_zero", 0x1780)),
    "f16": (("pos_zero", 0x0000), ("neg_zero", 0x8000), ("min_subnormal", 0x0001),
            ("max_subnormal", 0x03FF), ("neg_subnormal", 0x8003), ("min_normal", 0x0400),
            ("max_finite", 0x7BFF), ("neg_max_finite", 0xFBFF), ("pos_inf", 0x7C00),
            ("neg_inf", 0xFC00), ("qnan", 0x7E00), ("nan_payload", 0x7E25), ("neg_nan", 0xFE00),
            ("snan", 0x7C01)),
}
NONFINITE = ("pos_inf", "neg_inf", "qnan", "nan_payload", "neg_nan", "snan")

# fp32 masters at a half dtype's range limits: (name, fp32 bits, bf16 bits, f16 bits of
# round-to-nearest-even).  Overflow thresholds as in harness.SPECIAL_RECIPES, exact ties, and values
# below, at and above half of f16's smallest subnormal.
WRITE_BACK = (
    ("bf16_ovf_below", 0x7F7F7FFF, 0x7F7F, 0x7C00), ("bf16_ovf_at", 0x7F7F8000, 0x7F80, 0x7C00),
    ("bf16_ovf_above", 0x7F7F8001, 0x7F80, 0x7C00), ("neg_bf16_ovf_at", 0xFF7F8000, 0xFF80, 0xFC00),
    ("flt_max", 0x7F7FFFFF, 0x7F80, 0x7C00),
    ("f16_ovf_below", 0x477FEFFF, 0x4780, 0x7BFF), ("f16_ovf_at", 0x477FF000, 0x4780, 0x7C00),
    ("f16_ovf_above", 0x477FF001, 0x4780, 0x7C00), ("neg_f16_ovf_at", 0xC77FF000, 0xC780, 0xFC00),
    ("bf16_tie_down", 0x3F808000, 0x3F80, 0x3C04), ("bf16_tie_up", 0x3F818000, 0x3F82, 0x3C0C),
    ("f16_tie_down", 0x3F801000, 0x3F80, 0x3C00), ("f16_tie_up", 0x3F803000, 0x3F80, 0x3C02),
    ("f16_quarter_min_subnormal", 0x32800000, 0x3280, 0x0000),
    ("f16_half_min_subnormal", 0x33000000, 0x3300, 0x0000),
    ("f16_above_half_min_subnormal", 0x33000001, 0x3300, 0x0001),
    ("f16_subnormal_tie_up", 0x33C00000, 0x33C0, 0x0002),
    ("neg_f16_quarter_min_subnormal", 0xB2800000, 0xB280, 0x8000),
)
MASTER_CATALOGUE = (
    ("pos_zero", 0x00000000), ("neg_zero", 0x80000000), ("min_subnormal", 0x00000001),
    ("max_subnormal", 0x007FFFFF), ("neg_subnormal", 0x80000100), ("neg_flt_max", 0xFF7FFFFF),
    ("pos_inf", 0x7F800000), ("neg_inf", 0xFF800000), ("nan", 0x7FC00000),
    ("neg_nan_payload", 0xFFC01234),
    # fp32 subnormals that are bf16 rounding ties
    ("bf16_subnormal_tie_down", 0x00008000), ("bf16_subnormal_tie_up", 0x00018000),
) + tuple((name, b32) for name, b32, _, _ in WRITE_BACK)

# Optimizer state written after the first step: {key: fp32 bits}, keys the optimizer lacks are
# skipped, elements of an entry that leaves a key out keep their value.  BELOW / ABOVE put
# max_exp_avg_sq just below / above the exp_avg_sq the next step computes.
QNAN, INF, NINF = 0x7FC00000, 0x7F800000, 0xFF800000
BELOW, ABOVE = "below", "above"
STATE_CATALOGUE = (
    ("nan", dict(momentum_buffer=QNAN, exp_avg=QNAN, max_exp_avg_sq=QNAN)),
    ("nan_payload", dict(momentum_buffer=0x7FC0BEEF, exp_avg=0xFFC0BEEF,
                         max_exp_avg_sq=0x7FC0BEEF)),
    ("pos_inf", dict(momentum_buffer=INF, exp_avg=INF, exp_avg_sq=INF, max_exp_avg_sq=INF)),
    ("neg_inf", dict(momentum_buffer=NINF, exp_avg=NINF)),
    ("neg_zero", dict(momentum_buffer=0x80000000, exp_avg=0x80000000)),
    ("subnormal", dict(momentum_buffer=0x00000400, exp_avg=0x80000400, exp_avg_sq=0x00000400)),
    ("exp_avg_sq_zero", dict(exp_avg_sq=0)),
    ("max_below_new", dict(max_exp_avg_sq=BELOW)),
    ("max_above_new", dict(max_exp_avg_sq=ABOVE)),
)
STATE_KEYS = ("momentum_buffer", "exp_avg", "exp_avg_sq", "max_exp_avg_sq")

# Odd cycle lengths (coprime to 8 and to the chunk lengths), longer than their catalogues: element
# i of tensor t takes entry (i + SHIFT * t + STEP_SHIFT * step) % CYCLE, the randn background where
# that is past the catalogue's end.
CYCLE = {"g": 23, "w": 37, "s": 13}
SHIFT = {"g": 5, "w": 11, "s": 3}
STEP_SHIFT = 7
assert all(c % 2 == 1 for c in CYCLE.values()) and len(GRAD_CATALOGUE["bf16"]) < CYCLE["g"] and \
    len(MASTER_CATALOGUE) < CYCLE["w"] and len(STATE_CATALOGUE) < CYCLE["s"]

# (numel, parameter phase, gradient phase), phases in elements modulo 8 (16 bytes of a half dtype).
# Fresh fp32 state is 16-byte aligned, so the SGD / Adam kernels take vectors only where the
# parameter's phase is 0 or 4.
SEGMENTS = (
    (12 * CHUNK + 13, 4, 4),    # 13 chunks: a 4-element head, vectors (gradient aligned), a tail
    (12 * CHUNK + 13, 4, 1),    # the same with 8 scalar gradient loads per vector
    (2999, 3, 0),               # master phase differs from the parameter's: all scalar
    (2999, 2, 2),               # likewise
    (1, 0, 0), (7, 4, 6), (9, 0, 3),
)
SGD_PATHS = ("head", "vector_grad_aligned", "vector_grad_unaligned", "tail", "all_scalar")
# LAMB: the numel % 4 == 0 tensors take _foreach_norm's float4 accumulator mapping, the others the
# strided scalar one; a parameter 8-byte aligned at a chunk start takes the 4-wide apply.
LAMB_SEGMENTS = ((4000, 0, 0), (4000, 1, 3), (3001, 0, 0), (3001, 2, 1))
LAMB_PATHS = ("mapping_vector", "mapping_scalar", "apply_vector", "apply_scalar")


def _signed(values, width):
    return np.array(values, dtype={16: np.uint16, 32: np.uint32}[width]).view(
        {16: np.int16, 32: np.int32}[width])


class Layout:
    """Parameters as 1-D views of one flat half buffer and their gradients as views of another, at
    the phases of `segments`, with the catalogues they carry: `grads` [(name, half bits)], `masters`
    [(name, fp32 bits)] and `states` (a STATE_CATALOGUE or ())."""

    def __init__(self, dev, dtype, segments, seed, grads=(), masters=(), states=()):
        import torch
        self.dev, self.dtype = dev, dtype
        self.cat = {"g": tuple(grads), "w": tuple(masters), "s": tuple(states)}
        total = sum(n + 16 for n, _, _ in segments) + 16
        gen = torch.Generator(device=dev).manual_seed(seed)
        self.pflat = torch.randn(total, device=dev, generator=gen).to(dtype)
        self.gflat = torch.zeros(total, dtype=dtype, device=dev)
        self.params, self.grads = [], []
        po = go = 0
        for n, pph, gph in segments:
            po = -(-po // 8) * 8 + pph
            go = -(-go // 8) * 8 + gph
            self.params.append(torch.nn.Parameter(self.pflat[po:po + n]))
            self.grads.append(self.gflat[go:go + n])
            po, go = po + n, go + n
        self.tables = {"g": torch.tensor(_signed([b for _, b in grads] or [0], 16), device=dev),
                       "w": torch.tensor(_signed([b for _, b in masters] or [0], 32), device=dev)}

    def ids(self, kind, t, step=0, numpy=False):
        n = self.params[t].numel()
        shift = SHIFT[kind] * t + (STEP_SHIFT * step if kind == "g" else 0)
        if numpy:
            return (np.arange(n) + shift) % CYCLE[kind]
        import torch
        return (torch.arange(n, device=self.dev) + shift) % CYCLE[kind]

    def name(self, kind, t, i, step=0):
        k = int(self.ids(kind, t, step, numpy=True)[i])
        return self.cat[kind][k][0] if k < len(self.cat[kind]) else "randn"

    def fill_grads(self, step, gen, scale=1e-2):
        """randn * scale gradients with the gradient catalogue over them; sets every p.grad."""
        import torch
        for t, (p, g) in enumerate(zip(self.params, self.grads)):
            b = (torch.randn(g.numel(), device=self.dev, generator=gen) * scale).to(self.dtype)
            b = b.view(torch.int16)
            if self.cat["g"]:
                ids = self.ids("g", t, step)
                b = torch.where(ids < len(self.cat["g"]),
                                self.tables["g"][ids.clamp(max=len(self.cat["g"]) - 1)], b)
            g.copy_(b.view(self.dtype))
            p.grad = g
        return list(self.grads)

    def masters_for(self, t, current):
        """`current` (a master) with the master catalogue written over it."""
        import torch
        w = current.clone().view(torch.int32)
        if self.cat["w"]:
            ids = self.ids("w", t)
            w = torch.where(ids < len(self.cat["w"]),
                            self.tables["w"][ids.clamp(max=len(self.cat["w"]) - 1)], w)
        return w.view(torch.float32)

    def state_for(self, t, key, current, v_next=None):
        """`current` (state `key`) with the state catalogue written over it; v_next (float64) is the
        exp_avg_sq the next step computes, for BELOW / ABOVE."""
        import torch
        out = current.clone()
        ids = self.ids("s", t)
        for k, (_, values) in enumerate(self.cat["s"]):
            if key not in values:
                continue
            sel = ids == k
            v = values[key]
            if v in (BELOW, ABOVE):
                f = 1 - 2.0 ** -18 if v == BELOW else 1 + 2.0 ** -18
                out[sel] = (v_next * f).float()[sel]
            else:
                out.view(torch.int32)[sel] = int(_signed([v], 32)[0])
        return out


def describe(lay_of, params, opt, ref, bad, step):
    """The first differing elements of the first differing tensors, with what the catalogues put
    there."""
    import torch
    lines = []
    for i, k in bad[:4]:
        if k == "step":
            lines.append("tensor %d: step %r vs %r" % (i, opt.state[params[i]].get("step"),
                                                       ref.opt.state[ref.masters[i]].get("step")))
            continue
        pick = {"master": (opt.state[params[i]]["master_param"], ref.masters[i]),
                "param": (params[i], ref.params[i])}
        a, b = pick.get(k) or (opt.state[params[i]].get(k), ref.opt.state[ref.masters[i]].get(k))
        if a is None or b is None or a.shape != b.shape:
            lines.append("tensor %d %s: present / shape %s vs %s" % (
                i, k, None if a is None else tuple(a.shape), None if b is None else tuple(b.shape)))
            continue
        ba, bb = bits(a).reshape(-1), bits(b).reshape(-1)
        pos = (ba != bb).nonzero().flatten()
        mask = 0xFFFF if a.element_size() == 2 else 0xFFFFFFFF
        lines.append("tensor %d %s: %d of %d elements differ" % (i, k, pos.numel(), ba.numel()))
        lay, t = lay_of[i]
        g = bits(lay.grads[t]).reshape(-1)
        for j in pos[:6].tolist():
            lines.append("  [%d] ours 0x%x ref 0x%x | grad 0x%04x (%s) master %s state %s" % (
                j, int(ba[j]) & mask, int(bb[j]) & mask, int(g[j]) & 0xFFFF,
                lay.name("g", t, j, step), lay.name("w", t, j), lay.name("s", t, j)))
    return "\n".join(lines)


def assert_matches(opt, params, ref, lay_of, where, step):
    import torch
    torch.cuda.synchronize()
    bad = state_mismatches(opt, params, ref)
    assert not bad, "%s: %d tensors differ from the reference, first %s\n%s" % (
        where, len(bad), bad[:8], describe(lay_of, params, opt, ref, bad, step))


# ---- the kernels' path choice, restated ----------------------------------------------------------
def sgd_paths(p, g, state, n):
    """walk_chunk's split (csrc/optim.cu) of a segment into scalar head, 16-byte vectors (gradient
    aligned or not), scalar tail, or all scalar, from the data pointers: a label per element."""
    lab = np.empty(n, dtype=object)
    pp, gp = p.data_ptr(), g.data_ptr()
    for start in range(0, n, CHUNK):
        end = min(start + CHUNK, n)
        head = ((16 - ((pp + start * 2) & 15)) & 15) // 2
        vec = (pp & 1) == 0 and all(((s.data_ptr() + (start + head) * 4) & 15) == 0 for s in state)
        if not vec or head > end - start:
            head = end - start
        nvec = (end - start - head) // 8
        vbeg = start + head
        tail = vbeg + 8 * nvec
        lab[start:vbeg] = "head" if vec else "all_scalar"
        lab[vbeg:tail] = "vector_grad_aligned" if ((gp + vbeg * 2) & 15) == 0 else \
            "vector_grad_unaligned"
        lab[tail:end] = "tail"
    return [lab]


def lamb_paths(p, g, state, n):
    """lamb.cu's accumulator mapping (by numel % 4) and apply path (by the chunk-start alignment of
    master, moments and parameter) of every element."""
    mapping = np.full(n, "mapping_vector" if n % 4 == 0 else "mapping_scalar", dtype=object)
    apply = np.full(n, "apply_scalar", dtype=object)
    for start in range(0, n, NORM_CHUNK):
        m = min(NORM_CHUNK, n - start)
        if all(((s.data_ptr() + start * 4) & 15) == 0 for s in state) and \
                ((p.data_ptr() + start * 2) & 7) == 0:
            apply[start:start + 4 * (m // 4)] = "apply_vector"
    return [mapping, apply]


def check_coverage(opt, lays, paths, wanted, steps, kinds=("g", "w", "s")):
    """Every entry of every catalogue the layouts carry reaches every path in `wanted`, for the
    gradients at every step in `steps`."""
    restate = sgd_paths if paths == "sgd" else lamb_paths
    seen = {}
    for lay in lays:
        for t, (p, g) in enumerate(zip(lay.params, lay.grads)):
            st = opt.state[p]
            state = [st["master_param"]] + [st[k] for k in STATE_KEYS if k in st]
            for lab in restate(p, g, state, p.numel()):
                for kind in kinds:
                    if not lay.cat[kind]:
                        continue
                    for step in (steps if kind == "g" else (0,)):
                        ids = lay.ids(kind, t, step, numpy=True)
                        for path in wanted:
                            sel = ids[lab == path]
                            seen.setdefault((kind, step, path), set()).update(
                                sel[sel < len(lay.cat[kind])].tolist())
    sizes = {kind: max(len(lay.cat[kind]) for lay in lays) for kind in kinds}
    missing = {key: sorted(set(range(sizes[key[0]])) - ids) for key, ids in seen.items()
               if len(ids) < sizes[key[0]]}
    assert not missing, "catalogue entries that reach no element of a path: %s" % missing
    for kind in kinds:
        if sizes[kind]:
            assert all((kind, step if kind == "g" else 0, path) in seen
                       for path in wanted for step in (steps if kind == "g" else (0,))), kind


def write_state(opt, params, ref, lay_of, grads=None, betas=None):
    """The master and state catalogues, written into both sides; parameters become half(master)."""
    import torch
    with torch.no_grad():
        for i, p in enumerate(params):
            lay, t = lay_of[i]
            st, rst = opt.state[p], ref.opt.state[ref.masters[i]]
            w = lay.masters_for(t, st["master_param"])
            for dst in (st["master_param"], ref.masters[i], p, ref.params[i]):
                dst.copy_(w)
            if not lay.cat["s"]:
                continue
            for k in STATE_KEYS:
                if k not in st:
                    continue
                v_next = None
                if k == "max_exp_avg_sq":
                    g = grads[i].double()
                    v_next = st["exp_avg_sq"].double() * betas[1] + (1 - betas[1]) * g * g
                new = lay.state_for(t, k, st[k], v_next)
                st[k].copy_(new)
                rst[k].copy_(new)


def flatten(lays):
    params = [p for lay in lays for p in lay.params]
    lay_of = [(lay, t) for lay in lays for t in range(len(lay.params))]
    return params, lay_of


def sgd_layouts(dev, dtype, n=1, grads=True, masters=MASTER_CATALOGUE, states=STATE_CATALOGUE):
    return [Layout(dev, harness.torch_dtype(dtype), SEGMENTS, 10 + k,
                   grads=GRAD_CATALOGUE[dtype] if grads is True else grads, masters=masters,
                   states=states) for k in range(n)]


def run_edges(opt, ref, lays, paths, where, betas=None, after_first=None):
    """STEPS steps of both sides, catalogue gradients in every one, the master and state catalogues
    written after the first; everything compared after every step."""
    import torch
    params, lay_of = flatten(lays)
    sch = sched(opt)
    gen = torch.Generator(device=lays[0].dev).manual_seed(5)
    for step in range(STEPS):
        grads = [g for lay in lays for g in lay.fill_grads(step, gen)]
        if step == 1:
            check_coverage(opt, lays, paths, SGD_PATHS if paths == "sgd" else LAMB_PATHS,
                           range(STEPS))
            write_state(opt, params, ref, lay_of, grads, betas)
        opt.step()
        sch.step()
        ref.step(grads)
        assert_matches(opt, params, ref, lay_of, "%s step %d" % (where, step), step)
        if step == 0 and after_first is not None:
            after_first(params, opt)
    return params


# ---- 1. SGD --------------------------------------------------------------------------------------
SGD_HP = {"plain": dict(momentum=0.0),
          "momentum_wd_dampening": dict(momentum=0.9, weight_decay=1e-2, dampening=0.1),
          "nesterov_wd": dict(momentum=0.9, weight_decay=1e-2, nesterov=True),
          "dampening_one": dict(momentum=0.9, dampening=1.0),   # alpha 0: 0 * inf
          "lr_zero_group": dict(momentum=0.9)}


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("hp_id", list(SGD_HP))
def test_sgd_at_edge_values(tok_lib, hp_id, dtype):
    import torch
    from torch_on_k8s_b200.optim import MasterWeightSGD
    hp = SGD_HP[hp_id]
    lays = sgd_layouts(torch.device("cuda", 0), dtype, 2 if hp_id == "lr_zero_group" else 1)
    spec = [(lays[0].params, 0.1)] + [(lay.params, 0.0) for lay in lays[1:]]
    opt = MasterWeightSGD([dict(params=ps, lr=lr) for ps, lr in spec], lr=0.1, **hp)
    ref = Reference([(ps, dict(lr=lr)) for ps, lr in spec], stock("SGD", **hp))
    run_edges(opt, ref, lays, "sgd", "%s %s" % (hp_id, dtype))


# ---- 2. Adam / AdamW -----------------------------------------------------------------------------
ADAM_HP = {"adam_l2": ("Adam", dict(weight_decay=1e-2)),
           "adamw_negative_decay": ("AdamW", dict(weight_decay=1500.0)),   # 1 - lr * wd = -0.5
           "amsgrad": ("AdamW", dict(amsgrad=True, weight_decay=1e-2)),
           "betas_half": ("Adam", dict(betas=(0.5, 0.999))),                # lerp's branch boundary
           "betas_zero": ("Adam", dict(betas=(0.0, 0.0))),
           "eps_zero": ("Adam", dict(eps=0.0))}


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("hp_id", list(ADAM_HP))
def test_adam_at_edge_values(tok_lib, hp_id, dtype):
    import torch
    from torch_on_k8s_b200 import optim
    cls, hp = ADAM_HP[hp_id]
    lays = sgd_layouts(torch.device("cuda", 0), dtype)
    spec = [(lays[0].params, 1e-3)]
    opt = getattr(optim, "MasterWeight" + cls)([dict(params=ps, lr=lr) for ps, lr in spec],
                                               lr=1e-3, **hp)
    ref = Reference([(ps, dict(lr=lr)) for ps, lr in spec], stock(cls, **hp))
    zero_grad = []

    def first(params, opt):
        if hp_id != "eps_zero":
            return
        for p, (lay, t) in zip(params, flatten(lays)[1]):   # a zero gradient at step 1: 0 / 0
            g = bits(lay.grads[t]).reshape(-1)
            z = ((g == 0) | (g == -0x8000)).nonzero().flatten()
            w = opt.state[p]["master_param"].reshape(-1)[z]
            zero_grad.append((z.numel(), bool(w.isnan().all().item())))
    run_edges(opt, ref, lays, "sgd", "%s %s" % (hp_id, dtype), betas=hp.get("betas", (0.9, 0.999)),
              after_first=first)
    if hp_id == "eps_zero":
        assert sum(n for n, _ in zero_grad) > 0 and all(ok for _, ok in zero_grad), zero_grad


# ---- 3. LAMB -------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_lamb_at_edge_values(tok_lib, dtype):
    """The decay group mixes clean tensors with one NaN gradient element in the second of three
    chunks, one inf gradient element, a master whose square overflows and a master whose every
    square underflows (|w| = 0, ratio 1); the no-decay group carries the catalogues elementwise."""
    import torch
    from torch_on_k8s_b200.optim import MasterWeightLAMB
    dev = torch.device("cuda", 0)
    dt = harness.torch_dtype(dtype)
    nan_at, inf_at, big_at = NORM_CHUNK + 1234, 500, 7
    decay = Layout(dev, dt, ((2 * NORM_CHUNK + 4000, 0, 0), (1001, 1, 1), (2000, 0, 0), (513, 0, 0),
                             (1000, 0, 0), (4096, 3, 5)), 20)
    plain = Layout(dev, dt, LAMB_SEGMENTS, 21, grads=GRAD_CATALOGUE[dtype],
                   masters=MASTER_CATALOGUE, states=STATE_CATALOGUE)
    lays = [decay, plain]
    params, lay_of = flatten(lays)
    groups = [(decay.params, dict(lr=1e-3, weight_decay=WD)),
              (plain.params, dict(lr=5e-4, weight_decay=0.0))]
    opt = MasterWeightLAMB([dict(params=ps, **o) for ps, o in groups])
    ref = Reference(groups, RefLAMB)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(6)
    nd = len(decay.params)
    for step in range(STEPS):
        grads = decay.fill_grads(step, gen) + plain.fill_grads(step, gen)
        grads[0][nan_at] = float("nan")
        grads[1][inf_at] = float("inf")
        if step == 1:
            check_coverage(opt, [plain], "lamb", LAMB_PATHS, range(STEPS))
            write_state(opt, params[nd:], _Shifted(ref, nd), lay_of[nd:])
            with torch.no_grad():
                ws = [opt.state[params[2]]["master_param"].clone(),
                      opt.state[params[3]]["master_param"].clone()]
                ws[0][big_at] = 2.0 ** 64                        # its square overflows: |w| = inf
                u = torch.rand(ws[1].shape, device=dev, generator=gen) + 0.5
                ws[1] = torch.where(u > 1, u, -u) * 2.0 ** -80   # every square underflows: |w| = 0
                for i, w in zip((2, 3), ws):
                    for dst in (opt.state[params[i]]["master_param"], ref.masters[i], params[i],
                                ref.params[i]):
                        dst.copy_(w)
        opt.step()
        sch.step()
        ref.step(grads)
        assert_matches(opt, params, ref, lay_of, "%s step %d" % (dtype, step), step)
    assert params[0].numel() > 2 * NORM_CHUNK and NORM_CHUNK <= nan_at < 2 * NORM_CHUNK
    # the NaN gradient made only its own element NaN: every chunk took ratio 1, not NaN
    w = opt.state[params[0]]["master_param"]
    assert w.isnan().sum().item() == 1 and w[nan_at].isnan().item()


class _Shifted:
    """A view of a Reference from parameter `k` on, for write_state over one group's tensors."""

    def __init__(self, ref, k):
        self.opt, self.masters, self.params = ref.opt, ref.masters[k:], ref.params[k:]


# ---- 4. a clipped step after a non-finite total norm ---------------------------------------------
CLIP_CASES = {"sgd": ("SGD", dict(momentum=0.9, weight_decay=1e-2)),
              "adamw_amsgrad": ("AdamW", dict(amsgrad=True, weight_decay=1e-2)),
              "lamb": ("LAMB", {})}
CLIP = 1e-2
# step: (tensor, element, value); clip_grad_norm_'s coefficient becomes 0, then NaN
NONFINITE_STEPS = {1: (1, 11, float("inf")), 3: (2, 33, float("nan"))}


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("case", list(CLIP_CASES))
def test_clipped_step_after_nonfinite_norm(tok_lib, case, dtype):
    """error_if_nonfinite=False: an inf total norm scales every gradient by 0 (inf * 0 = NaN), a NaN
    one by NaN, and the optimizer steps anyway."""
    import torch
    from torch_on_k8s_b200 import optim
    dev = torch.device("cuda", 0)
    cls, hp = CLIP_CASES[case]
    lays = [Layout(dev, harness.torch_dtype(dtype), SEGMENTS[1:], 30)]
    params, lay_of = flatten(lays)
    if cls == "LAMB":
        groups = [(params[:3], dict(lr=1e-3, weight_decay=WD)),
                  (params[3:], dict(lr=1e-3, weight_decay=0.0))]
        opt = optim.MasterWeightLAMB([dict(params=ps, **o) for ps, o in groups], max_grad_norm=CLIP)
        ref = Reference(groups, RefLAMB, clip=CLIP)
    else:
        opt = getattr(optim, "MasterWeight" + cls)(params, lr=1e-3, max_grad_norm=CLIP, **hp)
        ref = Reference([(params, dict(lr=1e-3))], stock(cls, **hp), clip=CLIP)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(7)
    for step in range(5):
        grads = lays[0].fill_grads(step, gen)
        if step in NONFINITE_STEPS:
            t, i, v = NONFINITE_STEPS[step]
            grads[t][i] = v
        total = torch.nn.utils.get_total_norm([g.float() for g in grads])
        opt.step()
        sch.step()
        ret, _ = ref.step(grads)
        if cls != "LAMB":
            total = ret
        where = "%s %s step %d" % (case, dtype, step)
        assert_matches(opt, params, ref, lay_of, where, step)
        assert same_bits(opt.grad_norm, total), (where, opt.grad_norm, total)
        want = {1: torch.isinf, 3: torch.isnan}.get(step, torch.isfinite)
        assert want(total).item(), (where, total)


# ---- 5. unscaled steps at finite extremes --------------------------------------------------------
SCALED_CASES = {"sgd": ("SGD", dict(momentum=0.9, nesterov=True, weight_decay=1e-4)),
                "adamw_amsgrad": ("AdamW", dict(amsgrad=True)),
                "lamb": ("LAMB", {})}


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("case", list(SCALED_CASES))
def test_unscaled_step_at_finite_extremes(tok_lib, case, dtype):
    """Scaled gradients at the largest finite value, subnormals and +-0 (nothing non-finite, so no
    step is skipped) unscaled by 1 / (3 * 2^12) and later 1 / (3 * 2^13): the kUnscale kernels."""
    import torch
    from torch_on_k8s_b200 import optim
    dev = torch.device("cuda", 0)
    cls, hp = SCALED_CASES[case]
    finite = tuple(e for e in GRAD_CATALOGUE[dtype] if e[0] not in NONFINITE)
    segs = LAMB_SEGMENTS if cls == "LAMB" else SEGMENTS
    lays = [Layout(dev, harness.torch_dtype(dtype), segs, 40 + k, grads=finite) for k in range(2)]
    params, lay_of = flatten(lays)
    if cls == "LAMB":
        groups = [(lays[0].params, dict(lr=1e-3, weight_decay=WD)),
                  (lays[1].params, dict(lr=5e-4, weight_decay=0.0))]
        opt = optim.MasterWeightLAMB([dict(params=ps, **o) for ps, o in groups],
                                     loss_scale=new_loss_scale())
        ref = Reference(groups, RefLAMB, scale=(INIT_SCALE, INTERVAL))
    else:
        spec = [(lays[0].params, 1e-2), (lays[1].params, 5e-4)]
        opt = getattr(optim, "MasterWeight" + cls)([dict(params=ps, lr=lr) for ps, lr in spec],
                                                   lr=1e-2, loss_scale=new_loss_scale(), **hp)
        ref = Reference([(ps, dict(lr=lr)) for ps, lr in spec], stock(cls, **hp),
                        scale=(INIT_SCALE, INTERVAL))
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(8)
    scales = []
    for step in range(STEPS):
        grads = [g for lay in lays for g in lay.fill_grads(step, gen)]
        if step == 1:
            check_coverage(opt, lays, "lamb" if cls == "LAMB" else "sgd",
                           LAMB_PATHS if cls == "LAMB" else SGD_PATHS, range(STEPS), kinds=("g",))
        scales.append(opt.loss_scale.get_scale())
        opt.step()
        sch.step()
        where = "%s %s step %d" % (case, dtype, step)
        total, found = ref.step(grads)
        if cls == "LAMB":
            assert not found.item() and same_bits(opt.loss_scale.scale_tensor, ref.scaler._scale), \
                where
        else:
            assert not scaling_matches(opt, ref, found, total), where
        assert not opt.step_skipped, where
        assert_matches(opt, params, ref, lay_of, where, step)
    assert scales == [INIT_SCALE] * INTERVAL + [2 * INIT_SCALE], scales


# ---- 6. the half write-back at the range limits --------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("case", ["sgd", "adam", "lamb"])
def test_half_write_back_at_range_limits(tok_lib, case, dtype):
    """Masters at, just below and just above each overflow threshold and rounding tie, stepped by
    lr = 2^-100 (far below half an ulp of any of them): the parameters must be p.copy_(master), and
    the expected elements must have become +-inf or rounded to even."""
    import torch
    from torch_on_k8s_b200 import optim
    dev = torch.device("cuda", 0)
    lr = 2.0 ** -100
    masters = tuple((name, b32) for name, b32, _, _ in WRITE_BACK)
    want = {name: (bf if dtype == "bf16" else h) for name, _, bf, h in WRITE_BACK}
    segs = LAMB_SEGMENTS if case == "lamb" else SEGMENTS
    lays = [Layout(dev, harness.torch_dtype(dtype), segs, 50, masters=masters)]
    params, lay_of = flatten(lays)
    if case == "lamb":
        opt = optim.MasterWeightLAMB([dict(params=params, lr=lr, weight_decay=0.0)])
        ref = Reference([(params, dict(lr=lr, weight_decay=0.0))], RefLAMB)
    elif case == "adam":
        opt = optim.MasterWeightAdam(params, lr=lr)
        ref = Reference([(params, dict(lr=lr))], stock("Adam"))
    else:
        opt = optim.MasterWeightSGD(params, lr=lr)
        ref = Reference([(params, dict(lr=lr))], stock("SGD"))
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(9)
    written = None
    for step in range(3):
        grads = lays[0].fill_grads(step, gen)
        if step == 1:
            check_coverage(opt, lays, "lamb" if case == "lamb" else "sgd",
                           LAMB_PATHS if case == "lamb" else SGD_PATHS, (), kinds=("w",))
            write_state(opt, params, ref, lay_of)
            written = [bits(opt.state[p]["master_param"]).clone() for p in params]
        opt.step()
        sch.step()
        ref.step(grads)
        assert_matches(opt, params, ref, lay_of, "%s %s step %d" % (case, dtype, step), step)
    names = [name for name, _ in masters]
    for t, p in enumerate(params):
        ids = lays[0].ids("w", t)
        sel = ids < len(masters)
        w = bits(opt.state[p]["master_param"])
        assert torch.equal(w[sel], written[t][sel]), "a master at the limits moved (tensor %d)" % t
        got = bits(p)[sel].tolist()
        expect = [int(_signed([want[names[k]]], 16)[0]) for k in ids[sel].tolist()]
        wrong = [(names[k], hex(g & 0xFFFF), hex(e & 0xFFFF))
                 for k, g, e in zip(ids[sel].tolist(), got, expect) if g != e]
        assert not wrong, "tensor %d: %d parameters are not the rounded master, first %s" % (
            t, len(wrong), wrong[:5])
