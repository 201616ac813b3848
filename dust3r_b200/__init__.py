"""H100-native DUSt3R.  The view stage and the localisation step are exported lazily, so that importing the package (e.g.
`python -m dust3r_b200.build`) does not import torch."""

_VIEWS = ('prepare_views', 'prepare_batch', 'item_rng')
_LOCALIZATION = ('run_pnp', 'localize', 'get_pose_error', 'aggregate_stats')


def __getattr__(name):
    if name in _VIEWS:
        from . import views
        return getattr(views, name)
    if name in _LOCALIZATION:
        from . import localization
        return getattr(localization, name)
    raise AttributeError(f'module {__name__!r} has no attribute {name!r}')
