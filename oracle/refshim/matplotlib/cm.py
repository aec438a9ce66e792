"""Stand-in for matplotlib.cm (see the package docstring)."""
