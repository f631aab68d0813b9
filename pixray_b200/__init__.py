"""pixray_b200: H100-native engine for pixray's per-iteration hot path (see DESIGN.md).

`import pixray_b200 as pixray` exposes the reference's module-level calls (pixray.py:2005-2124): run, reset_settings,
add_settings, get_settings, apply_settings, do_init, do_run, add_custom_loss (pixray_b200/api.py)."""
__version__ = "0.1.0"

_API = ("run", "reset_settings", "add_settings", "get_settings", "apply_settings", "do_init", "do_run", "add_custom_loss",
        "get_image")


def __getattr__(name):
    if name in _API:
        from . import api
        return getattr(api, name)
    raise AttributeError(f"module 'pixray_b200' has no attribute '{name}'")
