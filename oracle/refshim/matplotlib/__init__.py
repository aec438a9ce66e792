"""Stand-in for matplotlib so the REFERENCE agent module (team_code_v2/lav_agent_fast.py imports matplotlib.cm for its
visualisation) can be imported by oracle/pin_control.py.  Test infrastructure only; nothing here is ever called."""
