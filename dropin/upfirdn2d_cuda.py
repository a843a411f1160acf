"""Import-time stand-in for the StyleGAN2 `upfirdn2d_cuda` extension.

`imaginaire.layers` hard-imports it (imaginaire/third_party/upfirdn2d/upfirdn2d.py:17) although no
SceneDreamer generator, trainer or config ever executes it.  With dropin/ on
PYTHONPATH the import resolves; any attempt to CALL into it fails loudly."""


def __getattr__(name):
    if name.startswith('__'):
        raise AttributeError(name)

    def _missing(*a, **k):
        raise RuntimeError('upfirdn2d_cuda.%s: this extension is not part of the SceneDreamer render path and is '
                           'not provided by scenedreamer_b200 (import-time stand-in only)' % name)
    return _missing
