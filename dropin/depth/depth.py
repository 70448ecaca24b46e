"""Stand-in for the original project's depth/depth.py. illustrip.py imports it at the top and calls it only with `--depth > 0`
(illustrip.py:277-278, 387-388, 396-397); the default `--depth 0` never reaches these names."""

REASON = ('aphantasia_b200: --depth > 0 is not supported. The depth warp runs a Depth Anything V2 model fetched through '
          'transformers, which this project does not provide; it is outside the optimisation hot path. Run with --depth 0.')


class InferDepthAny:
    def __init__(self, *args, **kwargs):
        raise NotImplementedError(REASON)


def depthwarp(*args, **kwargs):
    raise NotImplementedError(REASON)
