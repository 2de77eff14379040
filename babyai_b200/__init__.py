"""babyai_b200: a GPU-native (H100) batched BabyAI environment (the env hot path of
mila-iqia/babyai: MiniGridEnv.step/gen_obs, RoomGrid, RoomGridLevel, verifier,
ParallelEnv) behind the reference's own vectorised-env surface.

    from babyai_b200 import BabyAIVecEnv, ParallelEnv, ManyEnvs, make_envs
    from babyai_b200 import DeviceParallelEnv, ObssPreprocessor        # observations stay in HBM (learner.py)

The compute path is the CUDA library babyai_b200/libbabyai_b200.so (C ABI in
include/babyai_b200.h); there is no CPU fallback.
"""
from .levels import LEVELS, VOCAB, detokenize, level_spec  # noqa: F401


def __getattr__(name):
    # vecenv imports torch and loads the CUDA library: keep `import babyai_b200` light
    if name in ('BabyAIVecEnv', 'ParallelEnv', 'ManyEnvs', 'make_envs', 'EnvList', 'preprocess_obss', 'RGBImgPartialObsWrapper',
                'MODE_AUTORESET', 'MODE_FREEZE'):
        from . import vecenv
        return getattr(vecenv, name)
    if name in ('DeviceParallelEnv', 'DeviceManyEnvs', 'ObssPreprocessor', 'FixedVocabulary', 'ObsTensors', 'ObsBatch'):
        from . import learner
        return getattr(learner, name)
    if name in ('DemoRecorder', 'episodes_to_demos'):
        from . import demos
        return getattr(demos, name)
    if name in ('gymapi', 'evaluate'):
        import importlib
        return importlib.import_module('.' + name, __name__)
    raise AttributeError(name)
