"""Shared harness of the GEMM schedule tests: operands in padded layouts, launches into sentinel-filled buffers, and
bitwise comparison of their output windows."""
import torch

from _util import check_sentinel, sentinel_buffer, window

EPI = dict(STORE=0, GELU=1, SILU=2, GATE_RES=3, MUL_DGELU=4, F32_STORE=7)


def load_ops():
    """finetrainers_b200.ops, after checking that the library runs on this device."""
    from finetrainers_b200 import lib, ops
    lib.check(lib.load().b2d_device_check(), "device")
    return ops


def bits(t):
    """A bf16 or fp32 tensor's bit patterns, as integers of the same width."""
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def assert_same(got, want, what):
    """Two lists of tensors are equal bit for bit; a difference is reported at its first element."""
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        neq = bits(g) != bits(w)
        if neq.any():
            j = tuple(int(v) for v in neq.nonzero()[0])
            raise AssertionError(f"{what} [window {i}]: {int(neq.sum())} element(s) differ, first at {j}: "
                                 f"got {g[j].item()!r} want {w[j].item()!r}")


def _up8(x):
    return (x + 7) // 8 * 8


class Case:
    """Operands of one GEMM with every epilogue input it may use; launch() returns the output windows.

    Leading dimensions of out, out2, res and aux are N + 24, 40, 56 and 72.  Batch z reads rows z * 8 further down A (or
    columns of an MN-major A) and B rows / columns z * 16 further in, and writes out and out2 at z * c_boff, with
    40-element gaps between the slices.  The per-sample gates have samples of `rps` rows (default: all of M)."""

    def __init__(self, M, N, K, a_mn=False, b_mn=False, K2=0, group=0, batch=1, rps=None, seed=0):
        self.M, self.N, self.K, self.K2, self.group, self.batch = M, N, K, K2, group, batch
        self.a_mn, self.b_mn, self.rps = a_mn, b_mn, rps or M
        g = torch.Generator(device="cuda").manual_seed(seed)

        def rnd(r, c, s=1.0):
            return (torch.randn(r, _up8(c), device="cuda", generator=g) * s).bfloat16()

        z = batch - 1
        self.a_boff = (0, 8) if a_mn else (8, 0)
        self.b_boff = (0, 16) if b_mn else (16, 0)
        self.A = rnd(K, M + 8 * z) if a_mn else rnd(M + 8 * z, K)
        self.B = rnd(K, N + 16 * z, K ** -0.5) if b_mn else rnd(N + 16 * z, K, K ** -0.5)
        groups = (N + group - 1) // group if group else 1
        if K2:
            self.A2 = rnd(M, K2 * groups)
            self.B2 = rnd(K2, N, K2 ** -0.5) if b_mn else rnd(N, K2, K2 ** -0.5)
        self.bias = rnd(1, N)[0]
        self.ldc, self.ldc2, self.ldres, self.ldaux = N + 24, N + 40, N + 56, N + 72
        self.c_boff = M * self.ldc2 + 40 if batch > 1 else 0  # out and out2 share it
        self.res = rnd(M, self.ldres)
        self.aux = rnd(M, self.ldaux)
        # gate vectors of exactly N elements each; the temb rows hold gate then gate2, one row per sample
        self.tab = [rnd(1, N, 0.5)[0, :N].contiguous() for _ in range(2)]
        self.temb = rnd((M + self.rps - 1) // self.rps, 2 * N + 8, 0.5)

    def _buffer(self, ld, dtype):
        buf = sentinel_buffer((self.batch - 1) * self.c_boff + self.M * ld + 32, dtype)
        return buf, [window(buf, z * self.c_boff, self.M, self.N, ld) for z in range(self.batch)]

    def launch(self, ops, epi, out2=False, gate=False, gate2=False, in_place=False, bias=True, **launch):
        """One ops.gemm launch into fresh buffers: every batch's out window, then out2's.  gate2 writes its gated copy to
        out2, so it implies out2; in_place makes res the out buffer, holding the residual in its first window."""
        out2 = out2 or gate2
        buf, wins = self._buffer(self.ldc, torch.float32 if epi == "F32_STORE" else torch.bfloat16)
        kw = dict(M=self.M, N=self.N, K=self.K, ldc=self.ldc, a_mn=self.a_mn, b_mn=self.b_mn, batch=self.batch,
                  a_boff=self.a_boff, b_boff=self.b_boff, c_boff=self.c_boff, epi=EPI[epi], alpha=0.75,
                  bias=self.bias if bias else None, **launch)
        if self.K2:
            kw.update(A2=self.A2, B2=self.B2, K2=self.K2, a2_group_n=self.group)
        if epi == "GATE_RES":
            if in_place:
                wins[0].copy_(self.res[:, :self.N])
                kw.update(res=buf, ldres=self.ldc)
            else:
                kw.update(res=self.res, ldres=self.ldres)
            if gate or gate2:
                kw.update(temb_stride=self.temb.stride(0), rows_per_sample=self.rps)
            if gate:
                kw.update(gate_table=self.tab[0], gate_temb=self.temb)
            if gate2:
                kw.update(gate2_table=self.tab[1], gate2_temb=self.temb[:, self.N:])
        if epi == "MUL_DGELU":
            kw.update(aux=self.aux, ldaux=self.ldaux)
        if out2:
            buf2, wins2 = self._buffer(self.ldc2, torch.bfloat16)
            kw.update(out2=buf2, ldc2=self.ldc2)
        ops.gemm(self.A, self.B, buf, **kw)
        check_sentinel(buf, wins, f"{epi} out")
        if out2:
            check_sentinel(buf2, wins2, f"{epi} out2")
            wins += wins2
        return wins
