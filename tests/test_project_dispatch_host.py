"""CPU: the activated projection's symbol choice and argument layout (ops.project_activated_forward and
ops.project_activated_backward, shared by the autograd operators and SplatTrainer), recorded through a fake library
in every mode the trainer and the operators reach.  Each call is checked against a literal table, written out in the
argument order of the C ABI, and position by position against capi._SIGS."""
import ctypes as C

import pytest

from opensplat_b200 import capi, ops

# sentinel device addresses
M, S, Q, LG, SG, V, PJ, F3 = 0x1100, 0x1200, 0x1300, 0x1400, 0x1500, 0x1600, 0x1700, 0x1800   # SG: sigmoid(logits)
COV, XY, DE, RA, CO, NT, OP = 0x2100, 0x2200, 0x2300, 0x2400, 0x2500, 0x2600, 0x2700       # forward outputs
VXY, VDEP, VC, VO = 0x3100, 0x3200, 0x3300, 0x3400                                        # cotangents
GM, GSC, GQ, GL = 0x4100, 0x4200, 0x4300, 0x4400                                          # gradients
PART, CG0, CG1, ST = 0x5100, 0x5200, 0x5300, 0x5400                                       # ST: the stream
# distinct scalars
N, GLOB, FX, FY, CX, CY, H, W, TX, TY, CLIP = 1000, 1.25, 300.5, 301.5, 160.25, 120.75, 240, 320, 20, 15, 0.0125
K1, K2, K3, K4, TH = 0.015, -0.0025, 0.00035, -4.5e-05, 1.375
NBLOCKS = 4                  # ceil(N / 256), the rows of gsb_project_camera_partials_floats(N)
VD = object()                # the v_depth slot: VDEP or None


class _Buf:
    """A contiguous CUDA buffer as capi.ptr sees it, at a sentinel address."""
    is_cuda = True

    def __init__(self, addr, numel=0):
        self.addr, self._numel = addr, numel

    def is_contiguous(self):
        return True

    def data_ptr(self):
        return self.addr

    def numel(self):
        return self._numel


class _Lib:
    """Records (symbol, args) of every call and returns success."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        assert name in capi._SIGS, name

        def call(*args):
            self.calls.append((name, args))
            return 24 * NBLOCKS if name == "gsb_project_camera_partials_floats" else 0
        return call


MODES = {
    "pinhole": ops.ProjectionMode(),
    "pinhole_aa": ops.ProjectionMode(antialiased=True),
    "filter3d": ops.ProjectionMode(filter3d=_Buf(F3)),
    "filter3d_aa": ops.ProjectionMode(antialiased=True, filter3d=_Buf(F3)),
    "fisheye": ops.ProjectionMode(fisheye=(K1, K2, K3, K4, TH)),
    "fisheye_aa": ops.ProjectionMode(antialiased=True, fisheye=(K1, K2, K3, K4, TH)),
}

FORWARD = {
    "pinhole": ("gsb_project_forward_activated",
                (N, M, S, GLOB, Q, LG, V, PJ, FX, FY, CX, CY, H, W, TX, TY, CLIP, COV, XY, DE, RA, CO, NT, OP, ST)),
    "pinhole_aa": ("gsb_project_forward_activated_aa",
                   (N, M, S, GLOB, Q, LG, V, PJ, FX, FY, CX, CY, H, W, TX, TY, CLIP, COV, XY, DE, RA, CO, NT, OP, ST)),
    "filter3d": ("gsb_project_forward_activated_filter3d",
                 (N, M, S, GLOB, Q, LG, F3, V, PJ, FX, FY, CX, CY, H, W, TX, TY, CLIP, COV, XY, DE, RA, CO, NT, OP, 0,
                  ST)),
    "filter3d_aa": ("gsb_project_forward_activated_filter3d",
                    (N, M, S, GLOB, Q, LG, F3, V, PJ, FX, FY, CX, CY, H, W, TX, TY, CLIP, COV, XY, DE, RA, CO, NT, OP,
                     1, ST)),
    "fisheye": ("gsb_project_forward_fisheye",
                (N, M, S, GLOB, Q, LG, V, FX, FY, CX, CY, K1, K2, K3, K4, TH, H, W, TX, TY, CLIP, COV, XY, DE, RA, CO,
                 NT, OP, 0, ST)),
    "fisheye_aa": ("gsb_project_forward_fisheye",
                   (N, M, S, GLOB, Q, LG, V, FX, FY, CX, CY, K1, K2, K3, K4, TH, H, W, TX, TY, CLIP, COV, XY, DE, RA,
                    CO, NT, OP, 1, ST)),
}

# (mode, accumulate, camera gradient) -> the projection backward call; the pinhole projection without AA alone reads
# the saved sigmoid, every other mode the logits
BACKWARD = {
    ("pinhole", 0, 0): ("gsb_project_backward_activated",
                        (N, M, S, GLOB, Q, SG, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, ST)),
    ("pinhole", 1, 0): ("gsb_project_backward_activated_acc",
                        (N, M, S, GLOB, Q, SG, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, ST)),
    ("pinhole", 0, 1): ("gsb_project_backward_activated_camgrad",
                        (N, M, S, GLOB, Q, SG, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, 0, 0,
                         PART, ST)),
    ("pinhole", 1, 1): ("gsb_project_backward_activated_camgrad",
                        (N, M, S, GLOB, Q, SG, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, 1, 0,
                         PART, ST)),
    ("pinhole_aa", 0, 0): ("gsb_project_backward_activated_aa",
                           (N, M, S, GLOB, Q, LG, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, ST)),
    ("pinhole_aa", 1, 0): ("gsb_project_backward_activated_aa_acc",
                           (N, M, S, GLOB, Q, LG, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, ST)),
    ("pinhole_aa", 0, 1): ("gsb_project_backward_activated_camgrad",
                           (N, M, S, GLOB, Q, LG, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, 0, 1,
                            PART, ST)),
    ("pinhole_aa", 1, 1): ("gsb_project_backward_activated_camgrad",
                           (N, M, S, GLOB, Q, LG, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, 1, 1,
                            PART, ST)),
    ("filter3d", 0, 0): ("gsb_project_backward_activated_filter3d",
                         (N, M, S, GLOB, Q, LG, F3, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, 0, 0,
                          0, None, ST)),
    ("filter3d", 1, 0): ("gsb_project_backward_activated_filter3d",
                         (N, M, S, GLOB, Q, LG, F3, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, 1, 0,
                          0, None, ST)),
    ("filter3d", 0, 1): ("gsb_project_backward_activated_filter3d",
                         (N, M, S, GLOB, Q, LG, F3, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, 0, 0,
                          1, PART, ST)),
    ("filter3d", 1, 1): ("gsb_project_backward_activated_filter3d",
                         (N, M, S, GLOB, Q, LG, F3, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, 1, 0,
                          1, PART, ST)),
    ("filter3d_aa", 0, 0): ("gsb_project_backward_activated_filter3d",
                            (N, M, S, GLOB, Q, LG, F3, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, 0,
                             1, 0, None, ST)),
    ("filter3d_aa", 1, 0): ("gsb_project_backward_activated_filter3d",
                            (N, M, S, GLOB, Q, LG, F3, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, 1,
                             1, 0, None, ST)),
    ("filter3d_aa", 0, 1): ("gsb_project_backward_activated_filter3d",
                            (N, M, S, GLOB, Q, LG, F3, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, 0,
                             1, 1, PART, ST)),
    ("filter3d_aa", 1, 1): ("gsb_project_backward_activated_filter3d",
                            (N, M, S, GLOB, Q, LG, F3, V, PJ, FX, FY, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC, GQ, GL, 1,
                             1, 1, PART, ST)),
    ("fisheye", 0, 0): ("gsb_project_backward_fisheye",
                        (N, M, S, GLOB, Q, LG, V, FX, FY, K1, K2, K3, K4, TH, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC,
                         GQ, GL, 0, 0, None, ST)),
    ("fisheye", 1, 0): ("gsb_project_backward_fisheye",
                        (N, M, S, GLOB, Q, LG, V, FX, FY, K1, K2, K3, K4, TH, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC,
                         GQ, GL, 1, 0, None, ST)),
    ("fisheye", 0, 1): ("gsb_project_backward_fisheye",
                        (N, M, S, GLOB, Q, LG, V, FX, FY, K1, K2, K3, K4, TH, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC,
                         GQ, GL, 0, 0, PART, ST)),
    ("fisheye", 1, 1): ("gsb_project_backward_fisheye",
                        (N, M, S, GLOB, Q, LG, V, FX, FY, K1, K2, K3, K4, TH, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC,
                         GQ, GL, 1, 0, PART, ST)),
    ("fisheye_aa", 0, 0): ("gsb_project_backward_fisheye",
                           (N, M, S, GLOB, Q, LG, V, FX, FY, K1, K2, K3, K4, TH, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC,
                            GQ, GL, 0, 1, None, ST)),
    ("fisheye_aa", 1, 0): ("gsb_project_backward_fisheye",
                           (N, M, S, GLOB, Q, LG, V, FX, FY, K1, K2, K3, K4, TH, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC,
                            GQ, GL, 1, 1, None, ST)),
    ("fisheye_aa", 0, 1): ("gsb_project_backward_fisheye",
                           (N, M, S, GLOB, Q, LG, V, FX, FY, K1, K2, K3, K4, TH, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC,
                            GQ, GL, 0, 1, PART, ST)),
    ("fisheye_aa", 1, 1): ("gsb_project_backward_fisheye",
                           (N, M, S, GLOB, Q, LG, V, FX, FY, K1, K2, K3, K4, TH, H, W, RA, CO, VXY, VD, VC, VO, GM, GSC,
                            GQ, GL, 1, 1, PART, ST)),
}
PARTIALS_FLOATS = ("gsb_project_camera_partials_floats", (N,))
REDUCE = ("gsb_project_camera_grad_reduce", (NBLOCKS, PART, CG0, CG1, ST))


def _check_signature(name, args):
    """arity, and int / float / pointer (int or None) position by position, against capi._SIGS"""
    _, types = capi._SIGS[name]
    assert len(args) == len(types), name
    for i, (a, t) in enumerate(zip(args, types)):
        if t is C.c_void_p:
            assert a is None or type(a) is int, (name, i, a)
        elif t is C.c_float:
            assert type(a) is float, (name, i, a)
        else:
            assert t in (C.c_int, C.c_size_t) and type(a) is int, (name, i, a)


@pytest.mark.parametrize("mode", list(MODES))
def test_forward_symbol_and_arguments(mode):
    L = _Lib()
    ops.project_activated_forward(L, MODES[mode], N, _Buf(M), _Buf(S), GLOB, _Buf(Q), _Buf(LG), _Buf(V), _Buf(PJ), FX,
                                  FY, CX, CY, H, W, (TX, TY, 1), CLIP, tuple(map(_Buf, (COV, XY, DE, RA, CO, NT, OP))),
                                  ST)
    assert L.calls == [FORWARD[mode]]
    for name, args in L.calls:
        _check_signature(name, args)


@pytest.mark.parametrize("v_depth", [False, True])
@pytest.mark.parametrize("cam", ["off", "given", "allocated"])
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("mode", list(MODES))
def test_backward_symbol_and_arguments(mode, accumulate, cam, v_depth, monkeypatch):
    """cam: no camera gradient; the camera gradient into the caller's partial rows (SplatTrainer); or into rows
    allocated by the call, gsb_project_camera_partials_floats(n) floats (the autograd operators)."""
    allocated = []

    def empty(shape, dtype, like):
        allocated.append(shape)
        return _Buf(PART, shape[0])
    monkeypatch.setattr(ops, "_empty", empty)
    L = _Lib()
    kw = {}
    if cam != "off":
        kw["cam_grad"] = (_Buf(CG0), _Buf(CG1))
    if cam == "given":
        kw["cam_partials"] = _Buf(PART, 24 * NBLOCKS)
    ops.project_activated_backward(L, MODES[mode], N, _Buf(M), _Buf(S), GLOB, _Buf(Q), _Buf(LG), _Buf(SG), _Buf(V),
                                   _Buf(PJ), FX, FY, H, W, _Buf(RA), _Buf(CO), _Buf(VXY),
                                   _Buf(VDEP) if v_depth else None, _Buf(VC), _Buf(VO),
                                   tuple(map(_Buf, (GM, GSC, GQ, GL))), ST, accumulate=accumulate, **kw)
    name, args = BACKWARD[(mode, int(accumulate), int(cam != "off"))]
    want = [(name, tuple((VDEP if v_depth else None) if a is VD else a for a in args))]
    if cam == "allocated":
        want.insert(0, PARTIALS_FLOATS)
    if cam != "off":
        want.append(REDUCE)
    assert L.calls == want
    assert allocated == ([(24 * NBLOCKS,)] if cam == "allocated" else [])
    for name, args in L.calls:
        _check_signature(name, args)
