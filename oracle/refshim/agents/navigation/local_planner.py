"""Stand-in for agents.navigation.local_planner: the RoadOption enum of the CARLA 0.9.10 PythonAPI."""
import enum


class RoadOption(enum.Enum):
    VOID = -1
    LEFT = 1
    RIGHT = 2
    STRAIGHT = 3
    LANEFOLLOW = 4
    CHANGELANELEFT = 5
    CHANGELANERIGHT = 6
