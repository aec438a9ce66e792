"""Stand-in for the CARLA leaderboard package the REFERENCE agent module imports (its AutonomousAgent base class and the Track
enum), so oracle/pin_control.py can import team_code_v2/lav_agent_fast.py.  Test infrastructure only."""
