"""CPU checks of the tensor-core gradient program (query_jvp_kernel, mp_query_points_grad_mode in MP_MODE_TC), compiled
unmodified on the CPU model of tests/emu: against the reference's fp64 autograd goldens, its value against the tensor-core
query program bit for bit, across simulated SM counts and bulk-copy completion orders, outside the image, under the range
guard and with a device-side point count.  (Its ptxas report is checked with the rest of query_tc.cu in
test_ptxas_report.py.)"""
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import spec
from emu_harness import build, write_input
from grad_cases import GOLDEN_CASES, load_golden, load_grad_case, tc_bar


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return dict(jvp=build(tmp_path_factory, "emu_query_jvp_tc"), tc=build(tmp_path_factory, "emu_query_tc"))


def _write_input(path, c, n):
    write_input(path, c["feat"], c["points"][:, :, :n], c["calib"], c["proj"], c["chans"][-1], c["last_op"], c["Ws"], c["bs"])


def _run_jvp(emu, tmp_path, c, n, sms=3, env=None, tag="j"):
    """-> (value [Res,n], dpoints [3,n]) of the tensor-core gradient program"""
    res = c["chans"][-1]
    fin, fout = str(tmp_path / ("in_%s.bin" % tag)), str(tmp_path / ("out_%s.f32" % tag))
    _write_input(fin, c, n)
    args = [emu["jvp"], fin, fout, str(sms)]
    if c["grad_output"] is not None:
        fg = str(tmp_path / ("gout_%s.f32" % tag))
        c["grad_output"][:, :n].contiguous().numpy().astype(np.float32).tofile(fg)
        args.append(fg)
    r = subprocess.run(args, capture_output=True, text=True, timeout=3600, env=dict(os.environ, **(env or {})))
    assert r.returncode == 0 and "DEADLOCK" not in r.stderr, r.stderr[-2000:]
    out = torch.from_numpy(np.fromfile(fout, dtype=np.float32))
    assert out.numel() == (res + 3) * n
    return out[:res * n].reshape(res, n), out[res * n:].reshape(3, n)


def _run_tc(emu, tmp_path, c, n, env=None):
    """-> [Res,n] of the tensor-core query program"""
    fin, fout = str(tmp_path / "in_q.bin"), str(tmp_path / "out_q.f32")
    _write_input(fin, c, n)
    r = subprocess.run([emu["tc"], fin, fout, "3" if c["net"] == "G" else "0", "2"], capture_output=True, text=True,
                       timeout=3600, env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, r.stderr[-2000:]
    return torch.from_numpy(np.fromfile(fout, dtype=np.float32)).reshape(c["chans"][-1], n)


# ---- a torch restatement of the kernel's fp16 roundings ------------------------------------------------------------------
def _h(x):
    """round to fp16 (and back to float64)"""
    return x.to(torch.float16).to(torch.float64)


def tc_jvp_ref(feat, points, calib, Ws, bs, last_op, projection="orthogonal", z_scale=spec.Z_SCALE, grad_output=None):
    """The tensor-core gradient program restated in float64 with its fp16 roundings at the same places: the per-texel
    products (fp16 map, G0 = fp16(F16 . fp16(W0f)), S4 in full precision), the layer-0 chunk in fp16 arithmetic (one rounding
    per fused multiply-add, taps nw, ne, sw, se), the fp16 X operand and tangent rows, fp16 operands of layers 1-3 (W3 as
    the hi + lo pair for the colour head), the leaky-ReLU slope taken from the value's fp16 (layers 0-2) or full-precision
    (layer 3) pre-activation, and the layer-4 dot, S4 and the chain rule in full precision.  Only the order of the sums
    differs from the kernel.  feat [1,C,H,W]; points [1,3,N]; -> dpoints [3,N] (float64)."""
    f = feat[0].to(torch.float64)
    C, H, W = f.shape
    pts = points[0].to(torch.float64)
    cal = calib[0].to(torch.float64) if calib is not None else None
    xyz = spec.project_ref(pts, cal, projection)
    u, v, w = xyz[0], xyz[1], xyz[2]
    n = u.shape[0]
    in_img = (u >= -1) & (u <= 1) & (v >= -1) & (v <= 1)
    ix, iy = (u + 1) / 2 * (W - 1), (v + 1) / 2 * (H - 1)
    x0, y0 = torch.floor(ix), torch.floor(iy)
    x1, y1 = x0 + 1, y0 + 1
    okx0, okx1 = (x0 >= 0) & (x0 <= W - 1), (x1 >= 0) & (x1 <= W - 1)
    oky0, oky1 = (y0 >= 0) & (y0 <= H - 1), (y1 >= 0) & (y1 <= H - 1)
    cx0, cx1 = x0.clamp(0, W - 1).long(), x1.clamp(0, W - 1).long()
    cy0, cy1 = y0.clamp(0, H - 1).long(), y1.clamp(0, H - 1).long()
    off = [cy0 * W + cx0, cy0 * W + cx1, cy1 * W + cx0, cy1 * W + cx1]                      # nw, ne, sw, se
    ok = [okx0 & oky0, okx1 & oky0, okx0 & oky1, okx1 & oky1]
    wgt = [(x1 - ix) * (y1 - iy), (ix - x0) * (y1 - iy), (x1 - ix) * (iy - y0), (ix - x0) * (iy - y0)]
    dwx = [-(y1 - iy), y1 - iy, -(iy - y0), iy - y0]
    dwy = [-(x1 - ix), -(ix - x0), x1 - ix, ix - x0]
    wgt = [torch.where(ok[a], wgt[a], 0.0) for a in range(4)]
    dwx = [torch.where(ok[a] & in_img, dwx[a], 0.0) for a in range(4)]
    dwy = [torch.where(ok[a] & in_img, dwy[a], 0.0) for a in range(4)]
    zf = w * z_scale
    Wd = [x.to(torch.float64) for x in Ws]
    bd = [x.to(torch.float64) for x in bs]
    F = f.reshape(C, H * W).t()                                                             # [texel][C]
    F16 = _h(F)
    G0 = _h(F16 @ _h(Wd[0][:, :C]).t())                                                     # [texel][1024]
    S4 = F @ Wd[4][:, 128:128 + C].t()                                                      # [texel][R]
    # layer 0 in fp16 arithmetic
    acc = _h(_h(Wd[0][:, C])[None] * _h(zf)[:, None] + _h(bd[0])[None])
    for a in range(4):
        acc = _h(G0[off[a]] * _h(wgt[a])[:, None] + acc)
    s0 = torch.where(acc > 0, 1.0, spec.LEAKY_SLOPE)
    sl = _h(torch.tensor(spec.LEAKY_SLOPE, dtype=torch.float64))
    h0 = [torch.maximum(acc, _h(acc * sl))]
    h0.append(_h(sum(G0[off[a]] * dwx[a][:, None] for a in range(4)) * s0))
    h0.append(_h(sum(G0[off[a]] * dwy[a][:, None] for a in range(4)) * s0))
    h0.append(_h(_h(Wd[0][:, C])[None] * s0))
    X = [_h(sum(F16[off[a]] * wgt[a][:, None] for a in range(4))), _h(sum(F16[off[a]] * dwx[a][:, None] for a in range(4))),
         _h(sum(F16[off[a]] * dwy[a][:, None] for a in range(4))), torch.zeros(n, C, dtype=torch.float64)]

    def hidden(l, prev, fp16_out, pair=False):
        """layer l (1..3) on the 4 rows (value, ix, iy, zf): [prev | X] . W_l^T, then the epilogue"""
        hid = prev[0].shape[1]
        Wl = Wd[l][:, :hid + C]
        Wq = (_h(Wl) + _h(Wl - _h(Wl))) if pair else _h(Wl)
        pre = [torch.cat([prev[t], X[t]], 1) @ Wq.t() for t in range(4)]
        wz, b = Wd[l][:, hid + C][None], bd[l][None]
        val = pre[0] + (wz * zf[:, None] + b)
        if fp16_out:
            val = _h(val)
        s = torch.where(val > 0, 1.0, spec.LEAKY_SLOPE)
        outs = [torch.maximum(val, (_h(val * sl) if fp16_out else val * spec.LEAKY_SLOPE)), pre[1] * s, pre[2] * s,
                (pre[3] + wz) * s]
        return [_h(o) for o in outs] if fp16_out else outs

    h1 = hidden(1, h0, True)
    h2 = hidden(2, h1, True)
    h3 = hidden(3, h2, False, pair=Ws[4].shape[0] == 3)
    w4h, w4z, b4 = Wd[4][:, :128], Wd[4][:, 128 + C], bd[4]
    s4 = [sum(S4[off[a]] * wgt[a][:, None] for a in range(4)) + w4z[None] * zf[:, None] + b4[None],
          sum(S4[off[a]] * dwx[a][:, None] for a in range(4)), sum(S4[off[a]] * dwy[a][:, None] for a in range(4)),
          w4z[None].expand(n, -1)]
    y = [h3[t] @ w4h.t() + s4[t] for t in range(4)]                                         # [N][R]
    act = torch.sigmoid(y[0]) if last_op == spec.LAST_SIGMOID else torch.tanh(y[0])
    d = act * (1 - act) if last_op == spec.LAST_SIGMOID else 1 - act * act
    g = d * (grad_output.t().to(torch.float64) if grad_output is not None else 1.0)
    dix, diy, dzf = [(g * y[t]).sum(1) for t in (1, 2, 3)]
    du, dv, dw = dix * (W - 1) / 2, diy * (H - 1) / 2, dzf * z_scale
    if cal is None:
        gp = torch.stack([du, dv, dw])
    elif projection != "perspective":
        gp = cal[:3, :3].t() @ torch.stack([du, dv, dw])
    else:
        su, sv = du / w, dv / w
        gp = cal[:3, :3].t() @ torch.stack([su, sv, dw - su * u - sv * v])
    return torch.where(in_img[None], gp, 0.0)


@pytest.mark.parametrize("kind,name,n", GOLDEN_CASES)
def test_jvp_kernel_matches_reference_grad_golden(emu, tmp_path, kind, name, n):
    c = load_golden(kind, name)
    val, dp = _run_jvp(emu, tmp_path, c, n)
    assert (val - c["value"][:, :n]).abs().max().item() <= 1e-4
    ok, msg = tc_bar(dp, c["grad64"][:, :n], name)
    print(name, msg)
    assert ok, msg


@pytest.mark.parametrize("kind,name,n", GOLDEN_CASES)
def test_jvp_kernel_is_closer_to_its_fp16_restatement_than_the_restatement_to_fp64(emu, tmp_path, kind, name, n):
    """The kernel against tc_jvp_ref: the median and the 99th percentile of |kernel - restatement| are at most half those of
    |restatement - grad64|.  The restatement itself passes every golden's bar."""
    c = load_golden(kind, name)
    _, dp = _run_jvp(emu, tmp_path, c, n)
    ref = tc_jvp_ref(c["feat"], c["points"][:, :, :n], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"],
                     grad_output=c["grad_output"][:, :n] if c["grad_output"] is not None else None)
    g64 = c["grad64"][:, :n].to(torch.float64)
    ok, msg = tc_bar(ref, g64, name)
    assert ok, "restatement: " + msg
    k = (dp.double() - ref).abs().flatten()
    r = (ref - g64).abs().flatten()
    qk = [k.median().item(), torch.quantile(k, 0.99).item()]
    qr = [r.median().item(), torch.quantile(r, 0.99).item()]
    print(name, "|kernel - restatement| median %.2e p99 %.2e; |restatement - grad64| median %.2e p99 %.2e" % (*qk, *qr))
    assert qk[0] <= 0.5 * qr[0] and qk[1] <= 0.5 * qr[1], (qk, qr)


@pytest.mark.parametrize("name", ["g_persp", "c_rot"])
def test_jvp_value_is_the_tc_query_bit_for_bit(emu, tmp_path, name):
    c = load_grad_case(name)
    n = 40
    val, _ = _run_jvp(emu, tmp_path, c, n)
    assert torch.equal(val, _run_tc(emu, tmp_path, c, n))


def test_jvp_is_identical_on_1_to_3_sms_and_any_copy_order(emu, tmp_path):
    c = load_grad_case("g_nocalib")
    n = 50                    # 4 tiles of 16 points, the last one ragged
    want = _run_jvp(emu, tmp_path, c, n, sms=1, tag="s1")
    for sms, env in ((2, None), (3, None), (3, {"EMU_TC_ORDER": "random:7"}), (2, {"EMU_TC_ORDER": "random:3"})):
        got = _run_jvp(emu, tmp_path, c, n, sms=sms, env=env, tag="s%d" % sms)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), (sms, env)


def test_jvp_gradient_is_exactly_zero_outside_the_image(emu, tmp_path):
    c = load_grad_case("g_rot")
    n = 48
    val, dp = _run_jvp(emu, tmp_path, c, n)
    xyz = spec.project_ref(c["points"][0, :, :n], c["calib"][0])
    outside = ~((xyz[0] >= -1) & (xyz[0] <= 1) & (xyz[1] >= -1) & (xyz[1] <= 1))
    assert int(outside.sum()) >= 3
    assert bool((dp[:, outside] == 0).all()) and bool((val[:, outside] == 0).all())
    assert bool((dp[:, ~outside].abs().sum(0) > 0).all())


def test_jvp_range_guard_and_device_count(emu, tmp_path):
    """A launch guarded in range runs when the frame's max |feature| is at the limit and skips it when the limit is the
    float32 below (the tensor-core query skips exactly the same); the device-side count stops the launch at that point."""
    c = load_grad_case("g_nocalib")
    n = 40
    amax = c["feat"].abs().max().item()
    below = float(np.nextafter(np.float32(amax), np.float32(0)))
    full = _run_jvp(emu, tmp_path, c, n)
    at = _run_jvp(emu, tmp_path, c, n, env={"EMU_TC_LIMIT": repr(amax), "EMU_TC_GUARD": "1"}, tag="at")
    assert torch.equal(at[0], full[0]) and torch.equal(at[1], full[1])
    for guard, limit in (("1", below), ("2", amax)):
        env = {"EMU_TC_LIMIT": repr(limit), "EMU_TC_GUARD": guard}
        skipped = _run_jvp(emu, tmp_path, c, n, env=env, tag="sk" + guard)
        assert bool((skipped[0] == -4242).all()) and bool((skipped[1] == -4242).all()), guard
        assert bool((_run_tc(emu, tmp_path, c, n, env=env) == -4242).all()), guard
    k = 21
    cut = _run_jvp(emu, tmp_path, c, n, env={"EMU_COUNT": str(k)}, tag="cnt")
    assert torch.equal(cut[0][:, :k], full[0][:, :k]) and torch.equal(cut[1][:, :k], full[1][:, :k])
    assert bool((cut[0][:, k:] == -4242).all()) and bool((cut[1][:, k:] == -4242).all())

