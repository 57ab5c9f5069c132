"""Shared harness of the conv kernel tests (tests/test_conv_fwd_gpu.py, tests/test_conv_bwd_gpu.py): the library handle, a
Python mirror of conv_plan's tiling (csrc/conv_tc.cu), the profiler block that counts which of the library's kernels ran,
library options, exact and random operands, and sentinel-guarded NHWC channel slices."""
import collections

import torch

F64 = torch.float64
U = 2.0 ** -24
SENT16, SENT32 = 1000.0, -777.0
INVALID = -1


def L():
    from fasterseg_b200 import _lib
    return _lib.lib()


def _s():
    return torch.cuda.current_stream().cuda_stream


def _cpad(c):
    return (c + 7) // 8 * 8


def _out_size(H, W, k, s, p, dil, off):
    e = dil * (k - 1) + 1
    return (H - off[0] + 2 * p - e) // s + 1, (W - off[1] + 2 * p - e) // s + 1


# ---- conv_plan's tiling --------------------------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


N_TILES = (16, 32, 48, 64, 96, 128)


def tiling(Cout_t, Ho, Wo, N, sms=None):
    """conv_plan's tiling of a conv_tc problem with Cout_t output channels on N Ho x Wo maps ->
    dict(tw, th, tiles_w, tiles_h, m_tiles, n_tile, n_tiles, ctas); sms: the device's SM count unless given"""
    sms = _sms() if sms is None else sms
    npad = (Cout_t + 15) // 16 * 16
    tw = 16 if Wo >= 16 else 8
    th = 128 // tw
    tiles_w, tiles_h = -(-Wo // tw), -(-Ho // th)
    m_tiles = tiles_w * tiles_h * N
    n_tiles = -(-npad // 128)
    ni = 0
    while N_TILES[ni] * n_tiles < npad:
        ni += 1
    n_tiles = -(-npad // N_TILES[ni])
    while m_tiles * n_tiles < sms and ni > 0 and N_TILES[ni - 1] >= 32:
        ni -= 1
        n_tiles = -(-npad // N_TILES[ni])
    return dict(tw=tw, th=th, tiles_w=tiles_w, tiles_h=tiles_h, m_tiles=m_tiles, n_tile=N_TILES[ni], n_tiles=n_tiles,
                ctas=m_tiles * n_tiles)


RELU, AFFINE, FORCE_DIRECT, STATS, OUT_F32, X_DOWN2, Y_UP2 = 1, 2, 4, 8, 16, 64, 128   # fsb_conv_desc.flags


def _empty_plane(H, W, k, stride, pad, dil, off):
    """a stride-2 tap whose parity plane of x has no pixel (H or W of 1)"""
    if stride != 2:
        return False
    for r in range(k):
        for s in range(k):
            ph, pw = (r * dil - pad + off[0]) % 2, (s * dil - pad + off[1]) % 2
            if (H - ph + 1) // 2 <= 0 or (W - pw + 1) // 2 <= 0:
                return True
    return False


def fwd_plan(N, H, W, Cin, Cout, k, stride, pad, dil, off, x_cstride, flags, sms=None, tc2=-1):
    """conv_plan (csrc/conv_tc.cu) of an fsb_conv_fwd descriptor, FSB_CONV_TC2 = tc2 (-1 unset) -> dict(direct, Ho, Wo, and for
    conv_tc: win and the tiling).  H, W: the descriptor's (the half size with FSB_CONV_X_DOWN2)."""
    Ho, Wo = _out_size(H, W, k, stride, pad, dil, off)
    direct = bool(flags & FORCE_DIRECT) or Cin < 16 or x_cstride % 8 != 0 or k not in (1, 3) or stride not in (1, 2) or \
        _empty_plane(H, W, k, stride, pad, dil, off)
    if direct:
        return dict(direct=True, Ho=Ho, Wo=Wo)
    sms = _sms() if sms is None else sms
    t = tiling(Cout, Ho, Wo, N, sms)
    win_ok = k == 3 and stride == 1 and dil == 1 and tc2 != 0
    win = win_ok and ((t["ctas"] > sms and not flags & STATS) or tc2 == 1)
    return dict(t, direct=False, Ho=Ho, Wo=Wo, win=win)


def _n_tile(Cout_t, Ho, Wo, N):
    """conv_plan's output-channel tile for a conv_tc problem with Cout_t output channels on an Ho x Wo map"""
    return tiling(Cout_t, Ho, Wo, N)["n_tile"]


def _kernel_key(name):
    """profiler kernel name -> the key the expectations use: conv_tc instances by (n_tile, window, up2), the rest by name"""
    n = name.replace("void ", "").replace("fsb::", "").split("(")[0]
    for prefix, key in (("conv_tc_kernel<", "conv_tc"), ("conv_tc_up2_kernel<", "conv_tc_up2")):
        if n.startswith(prefix):
            bk, nt, win = [a.strip() for a in n[len(prefix):-1].split(",")]
            return "%s%s<%s>" % (key, "_win" if win == "true" else "", nt)
    return n


class Kernels:
    """counts the library's conv kernel launches of a block (torch.profiler; the weight packing the runs need is left out).
    CUPTI hands its activity records over in buffers, and a buffer can reach the profiler after the session that
    launched its kernels has ended, i.e. inside the next one.  So only the records of this block's own launches count: the
    kernels whose CUPTI correlation id belongs to a launch call made inside the block's time range.  `stale` counts the
    records of earlier launches that arrived here."""
    NAME = "conv_kernels"
    PACKING = ("pack_dgrad_kernel", "pack_conv_weight_kernel")

    def __enter__(self):
        from torch.profiler import ProfilerActivity, profile, record_function
        torch.cuda.synchronize()
        self.prof = profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA])
        self.prof.__enter__()
        self.mark = record_function(self.NAME)
        self.mark.__enter__()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.mark.__exit__(*exc)
        self.prof.__exit__(*exc)
        CUDA = torch.autograd.DeviceType.CUDA
        evs = list(self.prof.profiler.kineto_results.events())
        mark = [e for e in evs if e.name() == self.NAME and e.device_type() != CUDA]
        assert len(mark) == 1, "the block's annotation is missing from the trace"
        t0, t1 = mark[0].start_ns(), mark[0].end_ns()
        own = {e.correlation_id() for e in evs
               if e.device_type() != CUDA and e.name().startswith("cudaLaunchKernel") and t0 <= e.start_ns() <= t1}
        # the library launches through cudaLaunchKernelEx (cudaLaunchKernelExC in the trace): each of those launches of the
        # block must have its kernel record, none still in a CUPTI buffer
        lib = {e.correlation_id() for e in evs
               if e.device_type() != CUDA and e.name().startswith("cudaLaunchKernelExC") and t0 <= e.start_ns() <= t1}
        self.complete = lib <= {e.correlation_id() for e in evs if e.device_type() == CUDA}
        kernels = [e for e in evs if e.device_type() == CUDA and "fsb::" in e.name()]
        self.stale = sum(1 for e in kernels if e.correlation_id() not in own)
        self.counts = collections.Counter(_kernel_key(e.name()) for e in kernels
                                          if e.correlation_id() in own and not any(p in e.name() for p in self.PACKING))


def profiled(fn):
    """-> (fn(), Kernels of its launches).  A trace in which a launch of the block has no kernel record yet is incomplete: the
    block (fresh buffers, same inputs) is run again, at most three times in all."""
    for _ in range(3):
        with Kernels() as k:
            out = fn()
        if k.complete:
            return out, k
    raise AssertionError("the profiler's trace missed launches of the block three times")


def _assert_kernels(counts, expected):
    """exactly the expected launches of the library's kernels, by name"""
    expected = +collections.Counter(expected)
    assert dict(counts) == dict(expected), "kernels that ran %s, expected %s" % (dict(counts), dict(expected))


class Options:
    def __init__(self, opts):
        self.opts = opts

    def __enter__(self):
        from fasterseg_b200 import _lib
        self.saved = {k: _lib.get_option(k) for k in self.opts}
        for k, v in self.opts.items():
            _lib.set_option(k, v)

    def __exit__(self, *exc):
        from fasterseg_b200 import _lib
        for k, v in self.saved.items():
            _lib.set_option(k, v)


# ---- operands -------------------------------------------------------------------------------------------------------------------
def _ints(shape, gen):
    """sparse integers in {-1, 0, 1}: P(-1) = P(1) = 1/8"""
    v = torch.randint(0, 8, shape, generator=gen, device="cuda")
    return ((v == 1).to(torch.int8) - (v == 0).to(torch.int8)).to(F64)


def _normal(shape, gen):
    return torch.randn(shape, generator=gen, device="cuda", dtype=torch.float32).half().to(F64)


class Slice:
    """channels [off, off + C) of an NHWC buffer of pixel stride cs, with one spare pixel after the end"""

    def __init__(self, N, H, W, C, cs, off, dtype, fill_own, fill_other):
        self.shape, self.C, self.off = (N, H, W), C, off
        P = N * H * W
        self.flat = torch.full(((P + 1) * cs,), fill_other, dtype=dtype, device="cuda")
        self.buf = self.flat[:P * cs].view(N, H, W, cs)
        self.view = self.buf[..., off:off + C]
        if fill_own is not None:
            self.view.fill_(fill_own)

    def ptr(self):
        return self.view.data_ptr()

    def put(self, nchw):
        self.view.copy_(nchw.permute(0, 2, 3, 1).to(self.flat.dtype))
        return self

    def nchw(self):
        return self.view.permute(0, 3, 1, 2).to(F64)

    def bits(self):
        return self.flat.view(torch.int16 if self.flat.element_size() == 2 else torch.int32)


def _bits32(t):
    return t.view(torch.int32)


def _report(name, worst):
    print("%s worst err/bound: %s" % (name, ", ".join("%s %.3f" % kv for kv in sorted(worst.items()))))
    assert max(worst.values()) <= 1.0, worst
