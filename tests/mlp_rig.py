"""The harness of the MLP GPU suites (tests/test_gpu_mlp*.py): the fixtures, the input builders, one table of the C
heads (`Head`, as HeadKind in ktb_mlp.cu), the one place that lays out their arguments, a push rig, guarded buffers,
the guard-band driver and the status-case builders.  Not a test module: the suites import from it."""
import contextlib
import ctypes
import functools
from typing import Callable, NamedTuple

import pytest
import torch

import kubetorch_b200 as kt
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp, ops

SHIPPED_CHUNK = 16896          # ktb_set_tuning key 8 as the library ships it
NO_BIAS = (None, None, None)


# ---- fixtures and inputs ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def K():
    assert torch.cuda.is_available()
    L.load()
    ops.ensure_init([0])
    return ops


@contextlib.contextmanager
def tuning(chunk=None, stage_ce=None):
    """ktb_set_tuning key 8 (MLP rows per chunk) = chunk and key 22 (staged chunks pulled by copy engine) = stage_ce,
    each when given; both are back at the library's 16896 and 0 on exit."""
    try:
        if chunk is not None:
            ops.set_tuning(8, chunk)
        if stage_ce is not None:
            ops.set_tuning(22, stage_ce)
        yield
    finally:
        ops.set_tuning(8, SHIPPED_CHUNK)
        ops.set_tuning(22, 0)


@pytest.fixture
def chunk_rows(K, request):
    with tuning(chunk=request.param):
        yield request.param


CHUNKED = (256, 1024, 5 * 256 + 128)   # with ktb_set_tuning(8, 256): five whole chunks and a 128-row last chunk


def layer_cases(shapes):
    """(d_in, d_hidden, M, chunk_rows) parameters: every shape at the shipped chunk, and CHUNKED at 256-row chunks."""
    out = [pytest.param(*s, None, id=f"din{s[0]}-dh{s[1]}-M{s[2]}") for s in shapes]
    out.append(pytest.param(*CHUNKED, 256, id=f"din{CHUNKED[0]}-dh{CHUNKED[1]}-M{CHUNKED[2]}-chunk256"))
    return out


def randn(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).bfloat16()


def stream():
    return int(torch.cuda.current_stream(0).cuda_stream)


def ptr(t):
    return 0 if t is None else t.data_ptr()


def config(seed, d_out, bias=True):
    """(W1, W2, W3), (b1, b2, b3) of the config's policy (d_in 256, d_hidden 1024) with a head d_out wide."""
    w = (randn((1024, 256), seed, 0.02), randn((1024, 1024), seed + 1, 0.02), randn((d_out, 1024), seed + 2, 0.02))
    b = (randn((1024,), seed + 3, 0.1), randn((1024,), seed + 4, 0.1), randn((d_out,), seed + 5, 0.1)) if bias \
        else NO_BIAS
    return w, b


def policy_weights(golden, d_out):
    """The recorded policy weights with random biases; heads other than 64 wide are random too."""
    inp = golden["all_inputs"]
    g = torch.Generator().manual_seed(d_out)
    w1, w2 = inp["mlp_w1"], inp["mlp_w2"]
    w3 = inp["mlp_w3"] if d_out == 64 else (torch.randn(d_out, 1024, generator=g) * 0.02).bfloat16()
    b1, b2, b3 = ((torch.randn(n, generator=g) * 0.1).bfloat16() for n in (1024, 1024, d_out))
    return w1, b1, w2, b2, w3, b3


@contextlib.contextmanager
def deployed(fn, name, devices, **distribute):
    """`fn` deployed as `name` on Compute(gpus = the distinct devices) with one rank on each entry of `devices`; torn
    down on exit."""
    remote = kt.fn(fn, name=name).to(
        kt.Compute(gpus=len(set(devices)), allowed_serialization=["json", "pickle"]).distribute(
            "b200", workers=1, num_proc=len(devices), devices=list(devices), **distribute))
    try:
        yield remote
    finally:
        remote.teardown()


# ---- exact layers -----------------------------------------------------------------------------------------------------
def bf16(t):
    """fp64 → fp32 → bf16, each step round-to-nearest-even: a monotone rounding to bf16 (identical to direct RNE except
    where the fp64 value lies within fp32 rounding distance of a bf16 tie)."""
    return t.float().bfloat16().float()


def check_layer(got, a, b, bias, relu, what):
    """got[M, N] (bf16, from the kernel) must be act(a · bᵀ + bias) rounded to bf16 from SOME value that fp32
    accumulation of the exact bf16 × bf16 products (and the bias) could produce.  r = the exact result (fp64: every
    product is exact, the sum's error is far below the bound), e = n·2^-23·(Σ|a_k·b_k| + |bias|) a deliberately generous
    bound on the fp32 accumulation error of its n = K additions (K + 1 with a bias), and rounding is monotonic, so
    bf16(act(r − e)) <= got <= bf16(act(r + e)).  For almost every element that admits exactly one bf16 value: at least
    99.9 % must equal bf16(act(r))."""
    a64, b64 = a.double(), b.double()
    r = a64 @ b64.t()
    s = a64.abs() @ b64.abs().t()
    n = a.shape[1]
    if bias is not None:
        r = r + bias.double()
        s = s + bias.double().abs()
        n += 1
    e = (n * 2.0 ** -23) * s
    act = (lambda t: t.clamp_min(0)) if relu else (lambda t: t)
    g = got.float()
    lo, hi = bf16(act(r - e)), bf16(act(r + e))
    bad = ~((lo <= g) & (g <= hi))          # NaN fails too
    if bool(bad.any()):
        idx = bad.nonzero()[:6].tolist()
        rows = [(i, j, float(g[i, j]), float(lo[i, j]), float(hi[i, j]), float(r[i, j])) for i, j in idx]
        pytest.fail(f"{what}: {int(bad.sum())} of {g.numel()} outputs outside [bf16(act(r-e)), bf16(act(r+e))]; "
                    f"(row, col, got, lo, hi, r): {rows}")
    exact = float((g == bf16(act(r))).double().mean())
    print(f"{what}: {exact:.6f} of {g.numel()} outputs are the bf16 rounding of the fp64 result")
    assert exact >= 0.999, (what, exact)


def identity(n):
    return torch.eye(n, device="cuda").bfloat16()


def select(d_hidden, cols):
    """A head that copies hidden units `cols` to the logits: one product with 1.0, exact zeros elsewhere."""
    w = torch.zeros(len(cols), d_hidden, device="cuda")
    w[torch.arange(len(cols), device="cuda"), cols] = 1.0
    return w.bfloat16()


def copy_scales(d_in, d_hidden):
    """2^-(n // d_in) for every hidden unit n, exact (Python floats: a device pow need not be exact)."""
    return torch.tensor([2.0 ** -(n // d_in) for n in range(d_hidden)], dtype=torch.float64, device="cuda")


def scaled_copies(d_in, d_hidden):
    """W1[n, n mod d_in] = 2^-(n // d_in): h1 = exactly scaled copies of (non-negative) obs, distinct per K block."""
    n = torch.arange(d_hidden, device="cuda")
    w = torch.zeros(d_hidden, d_in, dtype=torch.float64, device="cuda")
    w[n, n % d_in] = copy_scales(d_in, d_hidden)
    return w.bfloat16()


def exact_h1(obs, d_in, d_hidden):
    """Non-negative obs through scaled_copies: h1 known exactly (power-of-two scaling of bf16 values)."""
    h1_exact = obs.double()[:, torch.arange(d_hidden, device="cuda") % d_in] * copy_scales(d_in, d_hidden)
    h1 = h1_exact.bfloat16()
    assert torch.equal(h1.double(), h1_exact)
    return h1


def hidden_through_head(obs, w1, w2, width, b1=None, b2=None):
    """The full hidden activation that the last layer sees, read out `width` units per call through a selection head:
    every column of every 256-wide tile (every epilogue register pair and lane group) is observed."""
    d_hidden = w1.shape[0]
    parts = [mlp.mlp_forward(obs, w1, w2, select(d_hidden, torch.arange(t * width, t * width + width, device="cuda")),
                             biases=(b1, b2, None))
             for t in range(d_hidden // width)]
    return torch.cat(parts, dim=1)


# ---- the heads and their arguments ------------------------------------------------------------------------------------
class Head(NamedTuple):
    """The C entries of one MLP head."""
    plain: str
    staged: str          # the plain entry itself when that takes the stage buffer (0: the plain form)
    pushed: str
    biases: bool         # b1, b2, b3 follow W1, W2, W3
    width: int           # the one head width the entries accept; 0: any from 1 to 256
    outputs: dict        # output -> its bytes per row, from d_out
    args: Callable       # named arguments -> the head's arguments, which sit between the weights and the scratch


def _policy_head(entry, outputs, args):
    return Head(entry, entry, entry + "_pushed", True, 0, outputs, args)


BIAS_FREE_64 = Head("ktb_mlp_bf16", "ktb_mlp_bf16_staged", "ktb_mlp_bf16_pushed", False, 64,
                    {"logits": lambda d: 2 * d}, lambda a: (a["logits"],))
GREEDY = _policy_head("ktb_mlp_bf16_policy", {"logits": lambda d: 2 * d, "actions": lambda d: 8},
                      lambda a: (a["logits"], a["actions"]))
SAMPLE = _policy_head("ktb_mlp_bf16_policy_sample", {"actions": lambda d: 8, "log_probs": lambda d: 4},
                      lambda a: (a["seed"], a["row_base"], a["actions"], a["log_probs"]))
GAUSSIAN = _policy_head("ktb_mlp_bf16_policy_gaussian", {"actions": lambda d: 4 * d, "log_probs": lambda d: 4},
                        lambda a: (a["log_std"], a["seed"], a["row_base"], a["actions"], a["log_probs"]))


def named_args(obs, w, b, out, seed=0, log_std=None, **more):
    """The named arguments of a plain call over all rows of obs with weights w and biases b (each may be None); `out`
    maps outputs to addresses (a missing output is not wanted); `more` adds or replaces arguments."""
    a = dict(obs=obs.data_ptr(), M=obs.shape[0], d_in=obs.shape[1], d_hidden=w[0].shape[0], d_out=w[2].shape[0],
             w1=w[0].data_ptr(), b1=ptr(b[0]), w2=w[1].data_ptr(), b2=ptr(b[1]), w3=w[2].data_ptr(), b3=ptr(b[2]),
             logits=0, actions=0, log_probs=0, seed=seed, row_base=0, log_std=ptr(log_std), stage=None,
             stream=stream())
    a.update(out)
    a.update(more)
    return a


def from_row(head, a, r0):
    """The named arguments `a` for the rows from r0 on: every output r0 rows further in, row_base r0 further."""
    out = {name: a[name] + r0 * row_bytes(a["d_out"]) if a[name] else 0 for name, row_bytes in head.outputs.items()}
    return dict(a, row_base=a["row_base"] + r0, **out)


def entry_args(head, a, push=False):
    """(entry, arguments...) of `head` on cuda:0 from the named arguments `a`: its pushed entry with `push`, else its
    plain entry, in the staged form when a["stage"] is not None."""
    weights = [a[k] for k in (("w1", "b1", "w2", "b2", "w3", "b3") if head.biases else ("w1", "w2", "w3"))]
    body = (a["M"], a["d_in"], a["d_hidden"], a["d_out"], *weights, *head.args(a), a["scratch"])
    if push:
        return (head.pushed, 0, a["stage"], a["stride"], *body, a["ctrl"], a["ctrl_root"], a["rank"], a["chunk_rows"],
                a["seq"], a["stream"])
    if a["stage"] is None and head.staged != head.plain:
        return (head.plain, 0, a["obs"], *body, a["stream"])
    return (head.plain if a["stage"] is None else head.staged, 0, a["obs"], *body, a["stage"] or 0, a["stream"])


# ---- guarded buffers, the push rig and the guard-band driver ----------------------------------------------------------
class Guarded:
    """An `nbytes` buffer, `offset` bytes past a 256-byte boundary, inside a larger allocation whose bands before and
    after hold a byte pattern: a write past the buffer lands in memory the test owns and shows up as a changed band.
    Each band is at least as large as the buffer (and at least 64 KiB), so even an overrun by a whole buffer stays
    inside memory the test owns."""

    FILL = 0xA5

    def __init__(self, nbytes, offset=0):
        self.nbytes = int(nbytes)
        band = max(1 << 16, (self.nbytes + 255) // 256 * 256)
        self.start = band + offset
        self.raw = torch.full((self.start + self.nbytes + band,), self.FILL, dtype=torch.uint8, device="cuda")

    def ptr(self):
        return self.raw.data_ptr() + self.start

    def view(self, dtype=torch.uint8):
        return self.raw[self.start:self.start + self.nbytes].view(dtype)

    def check(self, what):
        torch.cuda.synchronize()
        for name, band in (("before", self.raw[:self.start]), ("after", self.raw[self.start + self.nbytes:])):
            changed = (band != self.FILL).nonzero()
            assert changed.numel() == 0, f"{what}: {changed.numel()} bytes changed in the band {name} the " \
                                         f"{self.nbytes}-byte buffer (first at band offset {int(changed[0])})"


class PushRig:
    """What PushSession does for the MLP, for one head: ranks [0, 0, 0] on cuda:0 and ONE stream, the head's pushed
    entry on ranks 1.. and its plain entry on the root's shard.  Every flag a kernel waits on is published by work
    enqueued before it on that stream (or on library streams that stream already waits for), so no wait can block.
    Staging and scratch are guarded buffers of the documented sizes; `scratch_bytes(rows)` sizes a rank's scratch (the
    policy entries' by default).  The head's per-row inputs, `sides` ((name, bytes per row) in order), ride with the
    rows (ktb_push_scatter_ce_sides) into each staging half, laid out here and not by the package: the rows, then each
    side 8-byte aligned after the previous region, tighter than the package's 256-byte layout, since the pushed
    entries take any valid set of regions."""

    def __init__(self, K, M, d_in, d_hidden, chunk_rows, engine, head=None, n_ranks=3, sides=(), scratch_bytes=None):
        self.d_in, self.d_hidden, self.chunk_rows, self.engine, self.head = d_in, d_hidden, chunk_rows, engine, head
        self.n = n_ranks
        self.bounds = [K.shard_bounds(M, n_ranks, r) for r in range(n_ranks)]
        shard = max(e - b for b, e in self.bounds)
        end, self.offsets, self.row_bytes = shard * d_in * 2, {}, dict(sides)
        for name, row_bytes in sides:
            self.offsets[name] = (end + 7) // 8 * 8
            end = self.offsets[name] + shard * row_bytes
        self.stride = (end + 255) // 256 * 256
        self.ctrl = [torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda")
                     for _ in range(n_ranks)]
        self.stage = [None] + [Guarded(2 * self.stride) for _ in range(1, n_ranks)]
        size = scratch_bytes or (lambda rows: mlp.pushed_scratch_bytes(rows, d_hidden, chunk_rows))
        self.scratch = [None] + [Guarded(size(e - b)) for b, e in self.bounds[1:]]
        torch.cuda.synchronize()
        self.seq = 0

    def push(self, obs, sides, rank_entry, root_entry):
        """One call over the M rows of obs with the side tensors `sides` (by name): the scatter, then
        rank_entry(r, lo, hi, push) on ranks 1.., `push` holding the pushed entry's arguments (stage, stride, scratch,
        ctrl, ctrl_root, rank, chunk_rows, seq) and each side's offset by name, then root_entry(lo, hi, rows) on the
        root's shard, `rows` holding each side's address at row lo by name, then ktb_push_wait."""
        self.seq += 1
        seq, n, d_in, st = self.seq, self.n, self.d_in, stream()
        stage_ptrs = L.arr(ctypes.c_void_p, [0] + [s.ptr() for s in self.stage[1:]])
        ctrl_ptrs = L.arr(ctypes.c_void_p, [c.data_ptr() for c in self.ctrl])
        root = self.ctrl[0].data_ptr()
        names = list(self.offsets)
        if names:
            L.call("ktb_push_scatter_ce_sides", 0, obs.data_ptr(), obs.numel(), d_in, L.BF16, n, 0,
                   L.arr(ctypes.c_int, [0] * n), stage_ptrs, self.stride, ctrl_ptrs, root, self.chunk_rows * d_in,
                   len(names), L.arr(ctypes.c_void_p, [sides[k].data_ptr() for k in names]),
                   L.arr(ctypes.c_size_t, [self.row_bytes[k] for k in names]),
                   L.arr(ctypes.c_size_t, [self.offsets[k] for k in names]), seq, st)
        elif self.engine == "sm":
            L.call("ktb_push_scatter_chunked", 0, obs.data_ptr(), obs.numel(), d_in, L.BF16, n, 0, stage_ptrs,
                   self.stride, ctrl_ptrs, root, self.chunk_rows * d_in, 0, seq, st)
        else:
            L.call("ktb_push_scatter_ce", 0, obs.data_ptr(), obs.numel(), d_in, L.BF16, n, 0,
                   L.arr(ctypes.c_int, [0] * n), stage_ptrs, self.stride, ctrl_ptrs, root, self.chunk_rows * d_in,
                   seq, st)
        for r in range(1, n):
            lo, hi = self.bounds[r]
            rank_entry(r, lo, hi, dict(self.offsets, stage=self.stage[r].ptr(), stride=self.stride,
                                       scratch=self.scratch[r].ptr(), ctrl=self.ctrl[r].data_ptr(), ctrl_root=root,
                                       rank=r, chunk_rows=self.chunk_rows, seq=seq))
        lo, hi = self.bounds[0]
        root_entry(lo, hi, {k: sides[k].data_ptr() + lo * self.row_bytes[k] for k in names})
        L.call("ktb_push_wait", 0, root, n, 0, seq, st)

    def call(self, obs, w, b, out, seed=0, log_std=None, sides=None, **more):
        """One call of the head over the M rows of obs; `out` maps the head's outputs to the addresses of their M-row
        buffers, `sides` its side tensors by name, `more` adds named arguments (named_args)."""
        a = named_args(obs, w, b, out, seed, log_std, **more)

        def rank(r, lo, hi, push):
            L.call(*entry_args(self.head, dict(from_row(self.head, a, lo), M=hi - lo, **push), push=True))

        def root(lo, hi, rows):
            scratch = mlp._scratch_for(0, hi - lo, self.d_hidden)
            L.call(*entry_args(self.head, dict(from_row(self.head, a, lo), M=hi - lo, obs=a["obs"] + lo * self.d_in * 2,
                                               scratch=scratch.data_ptr(), **rows)))

        self.push(obs, sides or {}, rank, root)

    def statuses(self):
        out = []
        for c in self.ctrl:
            s = ctypes.c_uint(0)
            L.call("ktb_push_status", 0, c.data_ptr(), ctypes.byref(s))
            out.append(s.value)
        return out

    def check(self):
        """After the calls: every status 0, and no write past a rank's staging or scratch."""
        torch.cuda.synchronize()
        assert self.statuses() == [0] * self.n
        for r in range(1, self.n):
            self.stage[r].check(f"stage[{r}]")
            self.scratch[r].check(f"scratch[{r}]")


def run_guarded(form, head, K, chunk, obs, w, b, seed=0, log_std=None, offsets=None):
    """`head` over the M rows of obs with ktb_set_tuning(8, chunk), in `form`: "plain", "staged", or "pushed" (three
    calls of a PushRig with chunk_rows = 512 and the SM scatter, whose statuses must stay 0).  Every output of the head
    and every scratch and stage buffer is a Guarded buffer of the size include/ktb200.h documents; output `name` sits
    offsets[name] bytes past its 256-byte boundary.  Returns the buffers by name."""
    (M, d_in), d_hidden, d_out = obs.shape, w[0].shape[0], w[2].shape[0]
    bufs = {name: Guarded(M * row_bytes(d_out), (offsets or {}).get(name, 0))
            for name, row_bytes in head.outputs.items()}
    out = {name: buf.ptr() for name, buf in bufs.items()}
    with tuning(chunk):
        if form == "pushed":
            rig = PushRig(K, M, d_in, d_hidden, 512, "sm", head)
            for _ in range(3):
                rig.call(obs, w, b, out, seed, log_std)
            torch.cuda.synchronize()
            assert rig.statuses() == [0] * rig.n
            bufs.update({f"stage[{r}]": rig.stage[r] for r in range(1, rig.n)})
            bufs.update({f"scratch[{r}]": rig.scratch[r] for r in range(1, rig.n)})
            return bufs
        bufs["scratch"] = Guarded(L.load().ktb_mlp_scratch_bytes(M, d_hidden))
        if form == "staged":
            bufs["stage"] = Guarded(L.load().ktb_mlp_stage_bytes(M, d_in))
        L.call(*entry_args(head, named_args(obs, w, b, out, seed, log_std, scratch=bufs["scratch"].ptr(),
                                            stage=bufs["stage"].ptr() if form == "staged" else None)))
    return bufs


# ---- status cases -----------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _zero_buffers():
    """Zero buffers as large as any status case could use (d_in 512, d_out 512, fp32 actions 2048 × 512), kept for the
    session: an entry that took bad arguments would still write memory the tests own."""
    def zeros(n, dtype=torch.bfloat16):
        return torch.zeros(n, dtype=dtype, device="cuda")

    bias, scratch = zeros(1024), zeros(1 << 24, torch.uint8)
    ctrl = zeros(L.load().ktb_push_control_bytes(), torch.uint8)
    return dict(obs=zeros(2048 * 512), w1=zeros(1024 * 512), w2=zeros(1024 * 1024), w3=zeros(512 * 1024),
                b1=bias, b2=bias, b3=bias, logits=zeros(2048 * 512), actions=zeros(2048 * 512, torch.float32),
                log_probs=zeros(2048, torch.float32), log_std=zeros(512, torch.float32), scratch=scratch,
                stage=scratch, ctrl=ctrl, ctrl_root=ctrl)


def _status_args(head, defaults, overrides):
    z = _zero_buffers()
    a = {name: t.data_ptr() for name, t in z.items()}
    a.update(M=256, d_in=256, d_hidden=1024, d_out=head.width or 18, seed=1, row_base=0, stream=stream(), **defaults)
    for name, value in overrides.items():
        if name.endswith("_off"):
            name, value = name[:-4], z[name[:-4]].data_ptr() + value
        a[name] = value
    return a


def plain(head, **overrides):
    """(entry, arguments...) of `head`'s plain entry over the zero buffers: 256 rows, d_in 256, d_hidden 1024, the
    head's width or 18 outputs, seed 1.  An override replaces an argument by name, `<name>_off=k` points it k bytes
    into its buffer, and a stage (0 included) gives the staged form."""
    return entry_args(head, _status_args(head, dict(stage=None), overrides))


def pushed(head, **overrides):
    """As plain(), for `head`'s pushed entry as rank 1 of call 1: stage = the scratch buffer, stage_stride 1 MiB,
    chunk_rows 256."""
    return entry_args(head, _status_args(head, dict(stride=1 << 20, chunk_rows=256, rank=1, seq=1), overrides),
                      push=True)


def expect_status(args, status):
    with pytest.raises(L.KtbError) as ei:
        L.call(*args)
    assert ei.value.status == status, (args[0], str(ei.value))
    torch.cuda.synchronize()    # nothing was launched; the device stays healthy
