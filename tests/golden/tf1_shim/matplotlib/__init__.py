"""Import-time stand-in for matplotlib: ``examples/utilities.py`` imports ``ListedColormap`` for its
plotting helpers, which the fixture generators never call."""
