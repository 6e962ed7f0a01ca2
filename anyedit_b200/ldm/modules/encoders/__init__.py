"""Reference-path alias package (see anyedit_b200/__init__.py)."""
