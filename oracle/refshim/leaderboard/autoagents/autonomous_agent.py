"""Stand-in for leaderboard.autoagents.autonomous_agent: an empty AutonomousAgent base and the Track enum."""
import enum


class Track(enum.Enum):
    SENSORS = "SENSORS"
    MAP = "MAP"


class AutonomousAgent:
    pass
