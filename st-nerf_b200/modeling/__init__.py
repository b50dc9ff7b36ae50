"""Reference import name `modeling` (modeling/__init__.py:3-7) backed by the native renderer."""
from stnerf_b200.model import LayeredRFRender, build_layered_model

# demo/walking_demo.py:18 imports `build_model`, which the reference package does not define; export it so the
# demo imports (SURVEY section 2, row 20).
build_model = build_layered_model

__all__ = ["LayeredRFRender", "build_layered_model", "build_model"]
