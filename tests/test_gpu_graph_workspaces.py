"""GPU: CUDA graphs and the workspaces of the torch binding, judged against the float64 reference.

The backward and decode entry points take a scratch workspace, and the default backward also a zeroed one (its fp32 dq
accumulator), from a cache kept per (device, stream) that only grows; release_workspaces() empties it.  A captured
graph keeps raw pointers to the workspaces of the captured call and uses them at every replay, so a captured call owns
its workspaces.  A cached pair would go back to the allocator at the next growth or release while the graph still
points at it: the next tensor allocated on the stream would get the block and every replay would overwrite it (and
start dq from whatever it holds).

Every entry point that uses a workspace is captured, a lifetime event follows, and one replay on new inputs is judged:

  release   warm-up and capture on stream s, then release_workspaces()
  growth    warm-up and capture on s, then one eager call of a larger problem on s through the same entry point (and,
            after a captured decode step, a training step: decode shares the backward's scratch)
  cold      capture on a new stream with no warm-up, on memory filled with 0xFF; eager calls on that stream before the
            first replay and after it are judged too

After a release or growth, "bystanders" take every free block the allocator holds for s in its general pool, which is
where a freed workspace would be handed out next, and are filled with 0xFF.  After the replay: every output against
the float64 reference at C = 2 with the judges of the other GPU tests, bitwise equality with an eager call on the same
inputs where the route is reproducible (decode, the deterministic backward, o, dk and dv of the MHA default backward),
and every bystander still all 0xFF.  The replay runs only if the allocator has returned no memory to the driver since
the event, so a graph that points at a freed workspace fails by its values, never by a fault.

The last test replays a decode step and a training step captured one after the other on torch's default capture
stream concurrently, on two streams: each graph must have workspaces of its own."""
import os

import pytest
import torch

from elementwise_bounds import FMT, attention_bounds, check_bound, kernel_shift
from test_gpu_decode import make_cache, n_split_of
from test_gpu_decode_varlen import packed_split
from test_gpu_deterministic import bounded
from test_gpu_gqa import sm_count
from test_gpu_long_context import _fill_free_blocks, dense_scratch_bytes
from test_gpu_parity import TOL_OUT, bound_check, fcsa, record, rel_err  # noqa: F401
from test_gpu_varlen import cu_of, seq_check
from tile_ranges import group_split

_EXPANDABLE = "expandable_segments:true" in os.environ.get("PYTORCH_CUDA_ALLOC_CONF", "").replace(" ", "").lower()
pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(_EXPANDABLE, reason="written for the default allocator (no expandable segments)")]


def _randn(g, shape, dtype, amp=1.0):
    return (torch.randn(shape, generator=g) * amp).to(dtype)


# ---- the entry points ---------------------------------------------------------------------------------------------
class Train:
    """Forward + backward through autograd on static leaf tensors: dense (shapes (B, H, Hk, N, D)) or packed (lengths,
    with (H, Hk, D) of `small`).  Inputs are made on the host so that loading them into the statics allocates nothing
    on the device."""

    def __init__(self, dtype, small, big, bitwise, causal=True, deterministic=False, bias=False, lengths=None,
                 path=None):
        self.dtype, self.small, self.big, self.bitwise = dtype, small, big, bitwise
        self.causal, self.deterministic, self.bias, self.lengths, self.path = causal, deterministic, bias, lengths, path

    def inputs(self, seed, big=False):
        g = torch.Generator().manual_seed(seed)
        B, H, Hk, N, D = self.big if big and self.lengths is None else self.small
        if self.lengths is not None:
            ls = self.lengths[1 if big else 0]
            inp = dict(q=_randn(g, (sum(ls), H, D), self.dtype), k=_randn(g, (sum(ls), Hk, D), self.dtype),
                       v=_randn(g, (sum(ls), Hk, D), self.dtype), do=_randn(g, (sum(ls), H, D), self.dtype),
                       cu=cu_of(ls))
            inp["ls"] = ls
            return inp
        inp = dict(q=_randn(g, (B, H, N, D), self.dtype), k=_randn(g, (B, Hk, N, D), self.dtype),
                   v=_randn(g, (B, Hk, N, D), self.dtype), do=_randn(g, (B, H, N, D), self.dtype))
        if self.bias:
            inp["bias"] = _randn(g, (H, N, N), self.dtype)
        return inp

    def static(self, inp):
        st = {n: t.cuda() for n, t in inp.items() if torch.is_tensor(t)}
        for n in ("q", "k", "v", "bias"):
            if n in st:
                st[n].requires_grad_()
        st["ls"] = inp.get("ls")
        return st

    def load(self, st, inp):
        with torch.no_grad():
            for n, t in inp.items():
                if torch.is_tensor(t):
                    st[n].copy_(t)

    def run(self, st):
        import flash_cosine_sim_attention_b200 as pkg
        leaves = [st["q"], st["k"], st["v"]] + ([st["bias"]] if self.bias else [])
        if self.lengths is not None:
            m = max(st["ls"])
            o = pkg.flash_cosine_sim_attention_varlen(st["q"], st["k"], st["v"], st["cu"], st["cu"], m, m,
                                                      causal=self.causal, deterministic=self.deterministic)
        else:
            o = pkg.flash_cosine_sim_attention(st["q"], st["k"], st["v"], attn_bias=st.get("bias"), causal=self.causal,
                                               deterministic=self.deterministic)
        grads = torch.autograd.grad(o, leaves, st["do"])
        return dict(zip(("o", "dq", "dk", "dv", "d_bias"), (o.detach(),) + grads))

    def judge(self, got, inp, st):
        q, k, v, do = inp["q"], inp["k"], inp["v"], inp["do"]
        if self.lengths is not None:
            seq_check(self.dtype, tuple(got[n] for n in ("o", "dq", "dk", "dv")), q, k, v, do, inp["ls"], inp["ls"],
                      causal=self.causal)
        elif self.deterministic:
            bounded(self.dtype, got, q, k, v, do, causal=self.causal)
        else:
            bound_check(self.dtype, got, q, k, v, do, causal=self.causal, attn_bias=inp.get("bias"))

    def check_path(self, st):
        """The grouped-query split path: chosen by the library's rule and seen in the backward's launches."""
        if self.path != "split":
            return
        B, H, Hk, N, _ = self.small
        assert group_split(B, H, Hk, N, sm_count()) > 1
        import flash_cosine_sim_attention_b200 as pkg
        o = pkg.flash_cosine_sim_attention(st["q"], st["k"], st["v"], causal=self.causal)
        torch.cuda.synchronize()
        before = pkg.debug()
        torch.autograd.grad(o, (st["q"], st["k"], st["v"]), st["do"])
        torch.cuda.synchronize()
        assert pkg.debug() - before >= 5, "the grouped backward did not take the split path"


class Decode:
    """One decode step (append + attention over the cache) with split keys: dense new queries (B, H, n, D), or packed
    ones with a different count per sequence.  The caches are reset from the inputs at every load."""

    def __init__(self, dtype, packed, small, big):
        self.dtype, self.packed, self.small, self.big = dtype, packed, small, big
        self.bitwise = ("o",)

    def inputs(self, seed, big=False):
        H, Hk, D, cap, ns, lens = self.big if big else self.small
        g = torch.Generator().manual_seed(seed)
        B = len(lens)
        rows = (sum(ns),) if self.packed else (B,)
        tail = (D,) if self.packed else (ns[0], D)
        inp = dict(q=_randn(g, rows + (H,) + tail, self.dtype), k=_randn(g, rows + (Hk,) + tail, self.dtype),
                   v=_randn(g, rows + (Hk,) + tail, self.dtype))
        inp["kc"], inp["vc"] = make_cache(B, Hk, cap, D, self.dtype, lens, g, True, 1, 1.0)
        inp["seqlens"] = torch.tensor(lens, dtype=torch.int32)
        if self.packed:
            inp["cu"] = cu_of(ns)
        inp["ns"], inp["lens"], inp["cap"] = ns, lens, cap
        return inp

    def static(self, inp):
        st = {n: t.cuda().clone() for n, t in inp.items() if torch.is_tensor(t)}
        st["max_q"] = max(inp["ns"])
        return st

    def load(self, st, inp):
        for n, t in inp.items():
            if torch.is_tensor(t):
                st[n].copy_(t)

    def run(self, st):
        import flash_cosine_sim_attention_b200 as pkg
        kw = dict(cu_seqlens_q=st["cu"], max_seqlen_q=st["max_q"]) if self.packed else {}
        with torch.no_grad():
            o = pkg.flash_cosine_sim_attention_with_kv_cache(st["q"], st["kc"], st["vc"], st["seqlens"], st["k"],
                                                             st["v"], **kw)
        return {"o": o}

    def _seq(self, t, inp, b):
        """Sequence b of a per-row tensor as (1 or heads, rows, D) of the dense call."""
        if not self.packed:
            return t[b:b + 1]
        cu = inp["cu"].tolist()
        return t[cu[b]:cu[b + 1]].transpose(0, 1).unsqueeze(0)

    def judge(self, got, inp, st):
        """The append bitwise, then o of every sequence against the float64 reference on the operands the kernel read
        (test_gpu_decode.check_case, test_gpu_decode_varlen.run_packed)."""
        from flash_cosine_sim_attention_b200 import l2norm_tensors
        o, kc, vc = got["o"], st["kc"], st["vc"]
        q, k, v = (inp[n].cuda() for n in ("q", "k", "v"))
        kn, qh = l2norm_tensors(k)[0], l2norm_tensors(q)[0]
        exp_k, exp_v = inp["kc"].clone(), inp["vc"].clone()
        cap = inp["cap"]
        for b, L in enumerate(inp["lens"]):
            kb, vb = self._seq(kn, inp, b)[0], self._seq(v, inp, b)[0]
            n = max(0, min(kb.shape[1], cap - L))
            exp_k[b, :, L:L + n] = kb[:, :n]
            exp_v[b, :, L:L + n] = vb[:, :n]
        assert torch.equal(kc.view(torch.int16), exp_k.view(torch.int16)), "k_cache"
        assert torch.equal(vc.view(torch.int16), exp_v.view(torch.int16)), "v_cache"
        fmt = FMT[self.dtype]
        shift = kernel_shift(fmt, 8)
        for b, L in enumerate(inp["lens"]):
            qb, ob = self._seq(qh, inp, b), self._seq(o, inp, b)
            T = min(L + inp["ns"][b], cap)
            ref, bound = attention_bounds(qb, kc[b:b + 1, :, :T], vc[b:b + 1, :, :T], scale=8, causal=True,
                                          l2norm_qk=False, fmt=fmt, shift=shift, device="cuda")
            e = rel_err(ob, ref["o"].cpu().numpy())
            record(self.dtype, "graph decode o", e, TOL_OUT[self.dtype])
            assert e <= TOL_OUT[self.dtype], f"sequence {b} (L = {L}, T = {T}): {e}"
            record(self.dtype, "graph decode o/bound", check_bound("o", ob, ref, bound, fmt), 1.0)

    def check_path(self, st):
        H, Hk, D, cap, ns, lens = self.small
        if self.packed:
            assert packed_split(len(lens), H, Hk, max(ns), cap) > 1
        else:
            assert n_split_of(len(lens), H, Hk, ns[0], cap) > 1


ENTRIES = {
    "dense": Train(torch.bfloat16, (2, 4, 4, 300, 64), (4, 4, 4, 600, 64), ("o", "dk", "dv")),
    "gqa-split": Train(torch.float16, (2, 6, 2, 200, 128), (4, 6, 2, 400, 128), ("o",), path="split"),
    "bias": Train(torch.float16, (2, 3, 3, 150, 64), (4, 3, 3, 300, 64), ("o", "dk", "dv"), causal=False, bias=True),
    "deterministic": Train(torch.bfloat16, (2, 4, 2, 300, 64), (4, 4, 2, 600, 64), ("o", "dq", "dk", "dv"),
                           deterministic=True),
    "varlen": Train(torch.bfloat16, (1, 4, 4, 0, 64), None, ("o", "dk", "dv"),
                    lengths=([300, 0, 65, 129], [600, 0, 130, 258, 70])),
    "varlen-deterministic": Train(torch.bfloat16, (1, 4, 4, 0, 64), None, ("o", "dq", "dk", "dv"), deterministic=True,
                                  lengths=([300, 0, 65, 129], [600, 0, 130, 258, 70])),
    # (H, Hk, D, capacity, new tokens per sequence, cached lengths)
    "decode": Decode(torch.bfloat16, False, (8, 2, 64, 1024, [1, 1], [5, 700]),
                     (8, 2, 64, 2048, [4] * 6, [0, 5, 129, 700, 1500, 2044])),
    "packed-decode": Decode(torch.float16, True, (8, 2, 64, 1024, [1, 5, 3], [5, 300, 700]),
                            (8, 2, 64, 2048, [4, 16, 9, 1, 7, 30], [0, 5, 129, 700, 1500, 2000])),
}
# the training step after a captured decode step: more scratch than the decode step's split partials
TRAIN_AFTER_DECODE = Train(torch.bfloat16, (8, 8, 8, 1280, 64), None, ("o", "dk", "dv"))


# ---- allocator helpers --------------------------------------------------------------------------------------------
def _allocator_returns():
    """Counters that move when the allocator hands memory back to the driver (a block a graph points at could go)."""
    s = torch.cuda.memory_stats()
    return s.get("num_device_free", 0), s.get("num_alloc_retries", 0)


def _occupy(stream):
    """Bystanders: every inactive block of `stream` in the general pool taken back (ascending sizes, so best fit hands
    out exactly that block; small-pool blocks in pieces of at most 1 MB, as _fill_free_blocks does), filled with 0xFF
    and kept.  Best fit can give a piece part of another block and leave a block untaken, so this repeats until the
    pool holds no free block that a request could be handed (a large-pool block below 1 MB serves none)."""
    dev = torch.cuda.current_device()
    held = []
    with torch.cuda.stream(stream):
        for _ in range(8):
            sizes = []
            for seg in torch.cuda.memory_snapshot():
                if (seg["device"] != dev or seg["stream"] != stream.cuda_stream
                        or tuple(seg.get("segment_pool_id", (0, 0))) != (0, 0)):
                    continue
                for blk in seg["blocks"]:
                    if blk["state"] != "inactive":
                        continue
                    s = blk["size"]
                    if seg["segment_type"] == "small":
                        while s > 0:
                            sizes.append(min(s, 1 << 20))
                            s -= sizes[-1]
                    elif s >= 1 << 20:
                        sizes.append(s)
            if not sizes:
                break
            for s in sorted(sizes):
                t = torch.empty(s, dtype=torch.uint8, device="cuda")
                t.fill_(0xFF)
                held.append(t)
    return held


def _poison():
    """Fill the allocator's free memory with 0xFF (test_gpu_long_context.poison): what the capture allocates next comes
    from memory that reads as NaN."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    room = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
    del room
    _fill_free_blocks()


def _cached_bytes(run):
    """Bytes the workspace cache holds after `run` alone."""
    from flash_cosine_sim_attention_b200 import release_workspaces
    release_workspaces()
    run()
    torch.cuda.synchronize()
    return release_workspaces()


class Failures(list):
    """Every check of a test runs; the test fails at its end with all that went wrong."""

    def check(self, what, fn, *args):
        try:
            fn(*args)
        except AssertionError as e:
            self.append(f"{what}: {e}")

    def equal(self, what, got, want, names):
        for n in names:
            if not torch.equal(got[n], want[n]):
                self.append(f"{what}: {n} is not bitwise the eager call's")

    def done(self):
        assert not self, "\n".join(self)


# ---- release and growth -------------------------------------------------------------------------------------------
CASES = [(name, "release") for name in ENTRIES] + [(name, "growth") for name in ENTRIES] + [("decode", "growth-train")]


@pytest.mark.parametrize("name,event", CASES, ids=[f"{n}-{e}" for n, e in CASES])
def test_replay_after_lifetime_event(fcsa, name, event):
    entry = ENTRIES[name]
    big_entry = TRAIN_AFTER_DECODE if event == "growth-train" else entry
    fails = Failures()
    graph = None
    fcsa.release_workspaces()
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        inp0, inp = entry.inputs(seed=1), entry.inputs(seed=2)
        st = entry.static(inp0)
        if event != "release":
            big_inp = big_entry.inputs(seed=3, big=event == "growth")
            big_st = big_entry.static(big_inp)
            with torch.cuda.stream(s):
                small = _cached_bytes(lambda: entry.run(st))
                if event == "growth-train":
                    B, H, Hk, N, D = big_entry.small
                    grown = dense_scratch_bytes(big_entry.dtype, B, H, Hk, N, N, D) > small
                else:
                    grown = _cached_bytes(lambda: big_entry.run(big_st)) > small
            assert grown, "the larger call must grow the cached workspaces"
        with torch.cuda.stream(s):
            for _ in range(2):
                entry.run(st)                                      # warm-up: the stream's workspaces exist
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            out = entry.run(st)
        with torch.cuda.stream(s):
            if event == "release":
                fcsa.release_workspaces()
            else:
                big_got = big_entry.run(big_st)
            torch.cuda.synchronize()
            returns = _allocator_returns()
            bystanders = _occupy(s)
            entry.load(st, inp)
            assert _allocator_returns() == returns, \
                "the allocator returned memory to the driver after the event: not replaying"
            graph.replay()
            torch.cuda.synchronize()
            fails.check("replay", entry.judge, out, inp, st)
            eager = entry.run(st)
            torch.cuda.synchronize()
            fails.equal("replay", out, eager, entry.bitwise)
            if event != "release":
                fails.check("larger eager call", big_entry.judge, big_got, big_inp, big_st)
            hit = [t.numel() for t in bystanders if not bool((t == 0xFF).all())]
            if hit:
                fails.append(f"the replay wrote into {len(hit)} of {len(bystanders)} bystanders ({sum(hit)} bytes)")
            fails.check("path", entry.check_path, st)
        fails.done()
    finally:
        del graph
        torch.cuda.synchronize()
        fcsa.release_workspaces()


# ---- cold capture -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["dense", "varlen", "decode"])
def test_cold_capture(fcsa, name):
    """Capture on a stream nothing ran on, over memory that reads 0xFF: an eager call on that stream before the first
    replay must find a zeroed dq accumulator, and the replay and the eager call after it must be right too."""
    entry = ENTRIES[name]
    fails = Failures()
    graph = None
    fcsa.release_workspaces()
    try:
        inp0, inp1, inp2 = (entry.inputs(seed=seed) for seed in (4, 5, 6))
        st = entry.static(inp0)
        entry.run(st)                    # loads the kernels, on the current stream; its workspaces are released next
        torch.cuda.synchronize()
        fcsa.release_workspaces()
        _poison()
        s = torch.cuda.Stream()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            out = entry.run(st)
        with torch.cuda.stream(s):
            entry.load(st, inp1)
            first = entry.run(st)
            torch.cuda.synchronize()
            fails.check("eager call before the first replay", entry.judge, first, inp1, st)
            entry.load(st, inp2)
            graph.replay()
            torch.cuda.synchronize()
            fails.check("replay", entry.judge, out, inp2, st)
            after = entry.run(st)
            torch.cuda.synchronize()
            fails.check("eager call after the replay", entry.judge, after, inp2, st)
            fails.equal("replay", out, after, entry.bitwise)
        fails.done()
    finally:
        del graph
        torch.cuda.synchronize()
        fcsa.release_workspaces()


# ---- two graphs captured on one stream, replayed concurrently -------------------------------------------------------
def test_concurrent_replays_of_graphs_captured_on_one_stream(fcsa):
    """A decode step, then a smaller training step, both captured on torch's default capture stream; a cached workspace
    would be shared by the two (the training step needs no more scratch than decode).  One concurrent replay on two
    streams, both judged.  A race is not certain to show in one replay: this pins who owns what, run once."""
    dec, train = ENTRIES["decode"], Train(torch.bfloat16, (1, 2, 2, 128, 64), None, ("o", "dk", "dv"))
    fails = Failures()
    g1 = g2 = None
    fcsa.release_workspaces()
    try:
        d0, d1 = dec.inputs(seed=7), dec.inputs(seed=8)
        t0, t1 = train.inputs(seed=9), train.inputs(seed=10)
        dst, tst = dec.static(d0), train.static(t0)
        B, H, Hk, N, D = train.small
        assert dense_scratch_bytes(train.dtype, B, H, Hk, N, N, D) <= _cached_bytes(lambda: dec.run(dst))
        train.run(tst)                                               # loads the kernels
        torch.cuda.synchronize()
        fcsa.release_workspaces()
        g1, g2 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(g1):
            dout = dec.run(dst)
        with torch.cuda.graph(g2):
            tout = train.run(tst)
        dec.load(dst, d1)
        train.load(tst, t1)
        torch.cuda.synchronize()
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        for s, g in ((s1, g1), (s2, g2)):
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                g.replay()
        torch.cuda.synchronize()
        fails.check("decode replay", dec.judge, dout, d1, dst)
        fails.check("training replay", train.judge, tout, t1, tst)
        fails.done()
    finally:
        del g1, g2
        torch.cuda.synchronize()
        fcsa.release_workspaces()
