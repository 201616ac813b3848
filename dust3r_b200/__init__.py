"""H100-native DUSt3R.  The view stage is exported lazily, so that importing the package (e.g. `python -m dust3r_b200.build`)
does not import torch."""

_VIEWS = ('prepare_views', 'prepare_batch', 'item_rng')


def __getattr__(name):
    if name in _VIEWS:
        from . import views
        return getattr(views, name)
    raise AttributeError(f'module {__name__!r} has no attribute {name!r}')
