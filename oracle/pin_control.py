"""Pin the agent's decision tail (oracle/control_ref.py) against the REFERENCE and write tests/golden/agent_control.npz.  Every
other golden is left untouched.

Runs only where the reference sources are readable.  It imports the unmodified team_code_v2/pid.py and lav_agent_fast.py
(matplotlib, leaderboard.autoagents, agents.navigation and carla come from oracle/refshim) and
calls LAVAgent.pid_control and LAVAgent.plan_collide on a stub ``self`` per agent that holds what LAVAgent.setup gives them:
the config's attributes (:68-72) and two PIDControllers (:152-153).  It drives the seeded sequence of
oracle.control_ref.control_sequence (8 agents, 660 ticks: agents without and with 15 forecast rows, all six commands, NaN plans
and NaN forecast steps, one agent stopped throughout and one stopped for 620 ticks) through run_step's tail in its own order,
restated below with line citations, checks ControlTail against it and stores the seed and the reference's controls, flags and
counters per tick (the inputs are regenerated from the seed).

    python oracle/pin_control.py
"""
import json
import os
import sys
import types

import numpy as np
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("LAV_REFERENCE", "/root/reference")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "refshim"))
sys.path.insert(0, os.path.join(REF, "team_code_v2"))

from oracle.control_ref import (CONTROL_KEYS, CTL_BRAKE_MODEL, CTL_COLLIDE, CTL_CREEP, CTL_PID_BRAKE,  # noqa: E402
                                CTL_PLAN_INVALID, CTL_SPEED_CAP, ControlTail, control_sequence)

SEED, B, TICKS = 2024, 8, 660
STOPPED, HALTS = (2,), (3,)
GOLD = os.path.join(ROOT, "tests", "golden", "agent_control.npz")


def main():
    from lav_agent_fast import LAVAgent
    from pid import PIDController
    full = yaml.safe_load(open(os.path.join(REF, "team_code_v2", "config.yaml")))
    cfg = {k: full[k] for k in CONTROL_KEYS}
    agents = []
    for _ in range(B):
        s = types.SimpleNamespace(**cfg)                                                   # :71-72
        s.turn_controller = PIDController(K_P=cfg["turn_KP"], K_I=cfg["turn_KI"], K_D=cfg["turn_KD"], n=cfg["turn_n"])  # :152
        s.speed_controller = PIDController(K_P=cfg["speed_KP"], K_I=cfg["speed_KI"], K_D=cfg["speed_KD"], n=cfg["speed_n"])
        s.stop_counter, s.force_move = 0, 0                                                # :156-157
        agents.append(s)
    tail = ControlTail(B, cfg)
    control = np.zeros((TICKS, B, 3))
    flags = np.zeros((TICKS, B), dtype=np.int32)
    stop = np.zeros((TICKS, B), dtype=np.int64)
    force = np.zeros((TICKS, B), dtype=np.int64)
    worst = np.zeros(3)
    for tick, x in enumerate(control_sequence(SEED, B, TICKS, stopped=STOPPED, halts=HALTS)):
        for b, s in enumerate(agents):
            spd, cmd_value = float(x["speed"][b]), int(x["cmd"][b])
            if spd < 0.1:                                                                  # :228-231
                s.stop_counter += 1
            else:
                s.stop_counter = 0
            ego_plan_locs, ego_cast_locs = x["plan"][b], x["cast"][b]
            other_cast_locs, other_cast_cmds = x["other_locs"][b], x["other_cmds"][b]
            pred_bra = x["pred_bra"][b]
            if cmd_value in [4, 5]:                                                        # :325-326
                ego_plan_locs = ego_cast_locs
            f = 0
            for _ in range(2):                                                             # :328-336
                if not np.isnan(ego_plan_locs).any():
                    steer, throt, brake = LAVAgent.pid_control(s, ego_plan_locs, spd, cmd_value)
                else:
                    steer, throt, brake = 0, 0, 0
                    f = CTL_PLAN_INVALID
            f |= CTL_PID_BRAKE if brake else 0
            collide = LAVAgent.plan_collide(s, ego_plan_locs, other_cast_locs, other_cast_cmds)   # for every agent
            f |= (CTL_BRAKE_MODEL if float(pred_bra) > 0.1 else 0) | (CTL_COLLIDE if collide else 0)
            if float(pred_bra) > 0.1:                                                      # :340-343
                throt, brake = 0, 1
            elif collide:
                throt, brake = 0, 1
            if spd * 3.6 > s.max_speed:                                                    # :344-345
                throt = 0
                f |= CTL_SPEED_CAP
            if s.stop_counter >= 600:                                                      # :347-348
                s.force_move = 20
            if s.force_move > 0:                                                           # :350-352
                throt, brake = max(0.4, throt), 0
                s.force_move -= 1
                f |= CTL_CREEP
            control[tick, b] = steer, throt, brake
            flags[tick, b], stop[tick, b], force[tick, b] = f, s.stop_counter, s.force_move
        mine = tail.step(x["plan"], x["cast"], x["other_locs"], x["other_cmds"], x["pred_bra"], x["speed"], x["cmd"])
        assert np.array_equal(mine["flags"], flags[tick]), (tick, mine["flags"], flags[tick])
        assert np.array_equal(tail.stop, stop[tick]) and np.array_equal(tail.force, force[tick]), tick
        assert np.array_equal(mine["control"][:, 2], control[tick, :, 2]), tick
        worst = np.maximum(worst, np.abs(mine["control"] - control[tick]).max(0))
    print(f"ControlTail against the reference over {TICKS} ticks x {B} agents: flags, counters and brake equal; "
          f"max |steer| diff {worst[0]:.2e}, max |throttle| diff {worst[1]:.2e} (numpy {np.__version__})")
    assert worst.max() <= 1e-5
    counts = {name: int(((flags & bit) != 0).sum()) for name, bit in (("plan_invalid", CTL_PLAN_INVALID),
              ("pid_brake", CTL_PID_BRAKE), ("brake_model", CTL_BRAKE_MODEL), ("collide", CTL_COLLIDE),
              ("speed_cap", CTL_SPEED_CAP), ("creep", CTL_CREEP))}
    print("agent-ticks per flag:", counts)
    np.savez_compressed(GOLD, seed=SEED, batch=B, ticks=TICKS, stopped=np.array(STOPPED), halts=np.array(HALTS),
                        config=json.dumps(cfg), numpy_version=np.__version__, control=control, flags=flags, stop=stop,
                        force=force)
    print(f"wrote {GOLD} ({os.path.getsize(GOLD) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
