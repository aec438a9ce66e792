"""CPU: the numpy statement of the agent's decision tail (oracle/control_ref.py) — against the golden the reference itself wrote
(oracle/pin_control.py), on hand-built cases with known answers, and its summation order against numpy's own."""
import json
import os

import numpy as np
import pytest

from oracle.control_ref import (CTL_BRAKE_MODEL, CTL_COLLIDE, CTL_CREEP, CTL_PID_BRAKE, CTL_PLAN_INVALID, CTL_SPEED_CAP,
                                ControlTail, control_sequence, pairwise_sum)

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "agent_control.npz")
T, C = 20, 6


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def cfg(gold):
    return json.loads(str(gold["config"]))


def test_statement_equals_golden(gold, cfg):
    B, ticks = int(gold["batch"]), int(gold["ticks"])
    assert ticks > 650 and B == 8
    tail = ControlTail(B, cfg)
    seq = control_sequence(int(gold["seed"]), B, ticks, stopped=tuple(gold["stopped"]), halts=tuple(gold["halts"]))
    seen = set()
    for tick, x in enumerate(seq):
        r = tail.step(**x)
        np.testing.assert_array_equal(r["flags"], gold["flags"][tick], err_msg=f"tick {tick}")
        np.testing.assert_array_equal(tail.stop, gold["stop"][tick])
        np.testing.assert_array_equal(tail.force, gold["force"][tick])
        np.testing.assert_array_equal(r["control"][:, 2], gold["control"][tick, :, 2])
        np.testing.assert_allclose(r["control"][:, :2], gold["control"][tick, :, :2], rtol=0, atol=1e-5)
        seen.update(int(c) for c in x["cmd"])
        assert len(x["other_locs"][0]) == 0 and len(x["other_locs"][1]) == 15
    assert seen == set(range(C))
    for bit in (CTL_PLAN_INVALID, CTL_PID_BRAKE, CTL_BRAKE_MODEL, CTL_COLLIDE, CTL_SPEED_CAP, CTL_CREEP):
        assert ((gold["flags"] & bit) != 0).any(), bit


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_pairwise_order_is_numpys(dtype):
    rs = np.random.RandomState(3)
    for n in range(1, 129):
        x = (rs.randn(50, n) * rs.choice([1e-3, 1.0, 1e3], (50, n))).astype(dtype)
        mine = pairwise_sum(x)
        for i in range(50):
            assert mine[i].tobytes() == np.add.reduce(x[i]).tobytes(), (n, i)
            assert (mine[i] / dtype(n)).astype(dtype).tobytes() == x[i].mean().tobytes(), (n, i)


def test_degrees_is_one_product():
    x = np.random.RandomState(4).randn(100000) * 3
    assert np.array_equal(np.degrees(x), x * (180.0 / np.pi))


# ---- hand-built ticks --------------------------------------------------------------------------------------------------------
def line(step, T=T):
    """a straight plan driving forward (-y) ``step`` m per step, starting at the origin"""
    p = np.zeros((T, 2), np.float32)
    p[:, 1] = -step * np.arange(T, dtype=np.float32)
    return p


def one(tail, plan, rows=(), scores=None, pred_bra=0.0, speed=5.0, cmd=3, cast=None):
    rows = np.asarray(rows, np.float32).reshape(-1, C, T, 2)
    scores = np.ones((len(rows), C), np.float32) if scores is None else np.asarray(scores, np.float32).reshape(-1, C)
    cast = plan if cast is None else cast
    r = tail.step(plan[None], cast[None], [rows], [scores], np.float32([pred_bra]), np.float32([speed]), [cmd])
    return r["control"][0], int(r["flags"][0])


def static_row(x, y):
    """one forecast row whose branches all stand at (x, y)"""
    r = np.zeros((1, C, T, 2), np.float32)
    r[..., 0], r[..., 1] = x, y
    return r


def moving_row(plan, dx):
    """one forecast row whose branches follow the plan ``dx`` m to the side"""
    r = np.repeat(plan[None, None], C, 1).copy()
    r[..., 0] += np.float32(dx)
    return r


@pytest.mark.parametrize("d, hit", [(0.99, True), (1.01, False)])
def test_static_threshold(cfg, d, hit):
    _, f = one(ControlTail(1, cfg), line(0.5), static_row(d, -1.0))
    assert bool(f & CTL_COLLIDE) == hit


@pytest.mark.parametrize("d, hit", [(2.49, True), (2.51, False)])
def test_moving_threshold(cfg, d, hit):
    plan = line(0.5)
    _, f = one(ControlTail(1, cfg), plan, moving_row(plan, d))
    assert bool(f & CTL_COLLIDE) == hit


@pytest.mark.parametrize("y, hit", [(2.0, True), (np.nextafter(np.float32(2.0), np.float32(3.0)), False)])
def test_first_point_behind(cfg, y, hit):
    row = static_row(0.5, 0.0)
    row[0, 0, 0, 1] = y                           # the row's first point decides; y = 0.5 * ppm is not behind
    _, f = one(ControlTail(1, cfg), line(0.0), row)
    assert bool(f & CTL_COLLIDE) == hit


@pytest.mark.parametrize("score, hit", [(np.float32(0.2), True), (np.nextafter(np.float32(0.2), np.float32(0)), False)])
def test_score_threshold(cfg, score, hit):
    s = np.zeros((1, C), np.float32)
    s[0, 2] = score                               # 0.2f > 0.2: the branch counts
    _, f = one(ControlTail(1, cfg), line(0.5), static_row(0.5, -1.0), scores=s)
    assert bool(f & CTL_COLLIDE) == hit


@pytest.mark.parametrize("p, brakes", [(np.float32(0.1), True), (np.nextafter(np.float32(0.1), np.float32(0)), False)])
def test_brake_model_threshold(cfg, p, brakes):
    ctl, f = one(ControlTail(1, cfg), line(0.5), pred_bra=p, speed=1.0)
    assert bool(f & CTL_BRAKE_MODEL) == brakes    # 0.1f > 0.1
    assert (ctl[1] == 0.0 and ctl[2] == 1.0) if brakes else (ctl[1] > 0.0 and ctl[2] == 0.0)


def test_nan_step_in_branch(cfg):
    row = static_row(0.5, -1.0)
    _, f = one(ControlTail(1, cfg), line(0.5), row)
    assert f & CTL_COLLIDE
    row[0, :, 7, 0] = np.nan                      # every branch: np.min propagates the NaN, the branch never collides
    _, f = one(ControlTail(1, cfg), line(0.5), row)
    assert not f & CTL_COLLIDE
    row = static_row(0.5, -1.0)
    row[0, 1:, 7, 1] = np.nan                     # branch 0 stays clean and still collides
    _, f = one(ControlTail(1, cfg), line(0.5), row)
    assert f & CTL_COLLIDE


def test_nan_plan(cfg):
    tail = ControlTail(1, cfg)
    one(tail, line(0.5))
    turn, speed = tail.turn.copy(), tail.speed.copy()
    plan = line(0.5)
    plan[5, 0] = np.nan
    ctl, f = one(tail, plan, static_row(0.5, -1.0))
    assert f == CTL_PLAN_INVALID and ctl.tolist() == [0.0, 0.0, 0.0]
    np.testing.assert_array_equal(tail.turn, turn)
    np.testing.assert_array_equal(tail.speed, speed)
    ctl, f = one(tail, plan, static_row(0.5, -1.0), pred_bra=0.5)      # the brake rules still apply
    assert f == CTL_PLAN_INVALID | CTL_BRAKE_MODEL and ctl.tolist() == [0.0, 0.0, 1.0]


@pytest.mark.parametrize("cmd, valid", [(0, False), (1, False), (2, False), (3, False), (4, True), (5, True)])
def test_swap_for_lane_changes(cfg, cmd, valid):
    plan = line(0.5)
    plan[3, 1] = np.nan
    _, f = one(ControlTail(1, cfg), plan, cmd=cmd, cast=line(0.5))
    assert bool(f & CTL_PLAN_INVALID) != valid


def test_creep_after_600_stopped_ticks(cfg):
    tail = ControlTail(1, cfg)
    for i in range(599):
        ctl, f = one(tail, line(0.0), speed=0.0)
        assert not f & CTL_CREEP and ctl[1] == 0.0 and ctl[2] == 1.0
    for i in range(30):                           # re-armed every tick while the agent stays stopped
        ctl, f = one(tail, line(0.0), speed=0.0)
        assert f & CTL_CREEP and ctl.tolist()[1:] == [0.4, 0.0] and tail.force[0] == 19 and tail.stop[0] == 600 + i
    for i in range(19):                           # moving again: the last creep runs out
        ctl, f = one(tail, line(0.0), speed=0.5)
        assert f & CTL_CREEP and ctl[1] == 0.4 and tail.stop[0] == 0 and tail.force[0] == 18 - i
    ctl, f = one(tail, line(0.0), speed=0.5)
    assert not f & CTL_CREEP and ctl[1] == 0.0


@pytest.mark.parametrize("kmh, capped", [(35.05, True), (34.95, False)])
def test_speed_cap(cfg, kmh, capped):
    ctl, f = one(ControlTail(1, cfg), line(5.0), speed=kmh / 3.6)   # a plan fast enough to ask for throttle
    assert bool(f & CTL_SPEED_CAP) == capped
    assert (ctl[1] == 0.0) == capped


def test_double_pid_step(cfg):
    tail = ControlTail(1, cfg)
    plan = line(0.5)
    plan[:, 0] = 0.05 * np.arange(T, dtype=np.float32)          # aims to the right
    ctl, _ = one(tail, plan, speed=1.0)
    w = plan * np.float32(cfg["pixels_per_meter"])
    w[:, 1] = -w[:, 1]
    aim = w[cfg["aim_point"][3]]
    angle = np.degrees(np.pi / 2 - float(np.arctan2(np.float64(aim[1]), np.float64(aim[0])).astype(np.float32))) / 90
    n = cfg["turn_n"]
    assert tail.turn[0, -2:].tolist() == [angle, angle] and not tail.turn[0, :-2].any()
    mean = pairwise_sum(np.r_[np.zeros(n - 2), angle, angle]) / n
    want = cfg["turn_KP"] * angle + cfg["turn_KI"] * mean + cfg["turn_KD"] * 0.0      # the second step's derivative is 0
    assert ctl[0] == np.clip(want, -1.0, 1.0) and ctl[0] != 0.0
