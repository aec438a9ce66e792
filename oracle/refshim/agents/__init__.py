"""Stand-in for the CARLA PythonAPI ``agents`` package (team_code_v2/waypointer.py imports RoadOption from it), so
oracle/pin_control.py can import team_code_v2/lav_agent_fast.py.  Test infrastructure only."""
