"""Import-time stand-in for the StyleGAN2 `bias_act_cuda` extension.

`imaginaire.layers` hard-imports it (imaginaire/third_party/bias_act/bias_act.py:8) although no
SceneDreamer generator, trainer or config ever executes it.  With dropin/ on
PYTHONPATH the import resolves; any attempt to CALL into it fails loudly."""


def __getattr__(name):
    if name.startswith('__'):
        raise AttributeError(name)

    def _missing(*a, **k):
        raise RuntimeError('bias_act_cuda.%s: this extension is not part of the SceneDreamer render path and is '
                           'not provided by scenedreamer_b200 (import-time stand-in only)' % name)
    return _missing
