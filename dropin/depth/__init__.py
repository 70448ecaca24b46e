"""Drop-in `depth` package (illustrip.py:30 `from depth import depth`): the depth warp of `--depth > 0` is not provided."""
