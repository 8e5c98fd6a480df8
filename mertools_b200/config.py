"""Path dictionaries — same keys and meaning as MERBench/config.py:14-76 (PATH_TO_RAW_AUDIO,
PATH_TO_RAW_FACE, PATH_TO_TRANSCRIPTIONS, PATH_TO_FEATURES, PATH_TO_LABEL,
PATH_TO_PRETRAINED_MODELS).  The reference hard-codes one root per dataset; here the root comes from
the ``MER_DATA_ROOT`` environment variable (default ``./dataset``) and the per-dataset sub-layout is
the reference's.  A caller may also pass its own module with these attributes (every extractor takes
``config=``), which is how the reference's own ``config.py`` plugs in unchanged.
"""
import os

DATA_ROOT = os.environ.get("MER_DATA_ROOT", "./dataset")
DATASETS = ("MER2023", "IEMOCAPFour", "IEMOCAPSix", "CMUMOSI", "CMUMOSEI", "SIMS", "MELD", "SIMSv2")


def _root(ds):
    return os.path.join(DATA_ROOT, f"{ds.lower()}-dataset-process")


PATH_TO_RAW_AUDIO = {ds: os.path.join(_root(ds), "audio") for ds in DATASETS}
PATH_TO_RAW_FACE = {ds: os.path.join(_root(ds), "openface_face") for ds in DATASETS}
PATH_TO_TRANSCRIPTIONS = {ds: os.path.join(_root(ds), "transcription-engchi-polish.csv") for ds in DATASETS}
PATH_TO_FEATURES = {ds: os.path.join(_root(ds), "features") for ds in DATASETS}
# MERBench/config.py:64-73: IEMOCAP's two label sets are label_4way.npz / label_6way.npz (iemocap.py of the
# preprocessing writes both); here each has its own corpus root, where the reference shares one
_LABEL_FILES = {"MER2023": "label-6way.npz", "IEMOCAPFour": "label_4way.npz", "IEMOCAPSix": "label_6way.npz"}
PATH_TO_LABEL = {ds: os.path.join(_root(ds), _LABEL_FILES.get(ds, "label.npz")) for ds in DATASETS}
PATH_TO_PRETRAINED_MODELS = os.environ.get("MER_PRETRAINED_ROOT", "./tools")
