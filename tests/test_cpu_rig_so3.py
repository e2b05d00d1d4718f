"""A rig's joint SO(3) pre-alignment without a GPU: Context.rig passes joint_so3 into EfRigConfig, and ef_rig_create checks its
arguments before it needs a device."""
import ctypes

import numpy as np

EF_EINVAL = -1


class _FakeLib:
    """records the EfRigConfig ef_rig_create is given"""

    def __init__(self):
        self.cfg = None

    def ef_rig_create(self, ctx, cfg, out):
        from elasticfusion_b200 import capi

        self.cfg = capi.EfRigConfig.from_buffer_copy(ctypes.cast(cfg, ctypes.POINTER(capi.EfRigConfig)).contents)
        return 0


class _Handle:
    def __init__(self, value):
        self.h_cam = ctypes.c_void_p(value)


def test_context_rig_passes_joint_so3(monkeypatch):
    from elasticfusion_b200 import capi

    fake = _FakeLib()
    monkeypatch.setattr(capi, "lib", lambda: fake)
    ctx = capi.Context.__new__(capi.Context)
    ctx.h_ctx = ctypes.c_void_p(0x1000)
    cams = [_Handle(0x2000), _Handle(0x3000)]
    T = np.eye(4)
    T[:3, 3] = (0.1, 0.0, 0.0)
    for flag, want in ((False, 0), (True, 1)):
        capi.Context.rig(ctx, cams, [np.eye(4), T], joint_so3=flag)
        assert fake.cfg.joint_so3 == want and fake.cfg.n == 2
        assert np.array_equal(np.array(fake.cfg.T_0i[1][:]).reshape(4, 4), T)
    capi.Context.rig(ctx, cams)
    assert fake.cfg.joint_so3 == 0


def test_rig_create_rejects_null_context_with_joint_so3():
    from elasticfusion_b200 import capi

    cfg = capi.EfRigConfig()
    cfg.n = 1
    cfg.T_0i[0][:] = np.eye(4).reshape(16).tolist()
    cfg.joint_so3 = 1
    rig = ctypes.c_void_p()
    assert capi.lib().ef_rig_create(None, ctypes.byref(cfg), ctypes.byref(rig)) == EF_EINVAL
