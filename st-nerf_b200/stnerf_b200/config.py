"""cfg stub for hosts without yacs: the fields `LayeredRFRender.__init__` reads (modeling/layered_rfrender.py:23-37),
with the shipped configs' values (configs/config_taekwondo.yml:51-66), plus the two knobs of the native path."""
import types


def make_cfg(layer_num, n1, n2, use_space_time, precision="exact", chunk_rays=0):
    M = types.SimpleNamespace(
        BOARDER_WEIGHT=1e10, SAMPLE_METHOD="BBOX", SAME_SPACENET=False, TKERNEL_INC_RAW=True,
        POSE_REFINEMENT=False, USE_DIR=True, USE_DEFORM_VIEW=False, USE_DEFORM_TIME=True,
        USE_SPACE_TIME=use_space_time, BKGD_USE_DEFORM_TIME=False, BKGD_USE_SPACE_TIME=False,
        DEEP_RGB=False, COARSE_RAY_SAMPLING=n1, FINE_RAY_SAMPLING=n2, B200_PRECISION=precision,
        B200_CHUNK_RAYS=chunk_rays)
    return types.SimpleNamespace(MODEL=M, DATASETS=types.SimpleNamespace(LAYER_NUM=layer_num))


def make_render_cfg(output_dir, dataset_dir, layer_num, frame_num, size_test, n1=64, n2=128, use_space_time=True,
                    frame_offset=0, scale=1.0, fixed_near=-1.0, fixed_far=-1.0, precision="exact", original_size=None):
    """cfg for `render.LayeredNeuralRenderer`: `make_cfg` plus the dataset / output fields of configs/config_*.yml
    (OUTPUT_DIR, DATASETS.TRAIN/FRAME_NUM/FRAME_OFFSET/SCALE/FIXED_NEAR/FIXED_FAR/CAMERA_NUM, INPUT.SIZE_TEST)."""
    cfg = make_cfg(layer_num, n1, n2, use_space_time, precision)
    cfg.OUTPUT_DIR = output_dir
    D = cfg.DATASETS
    D.TRAIN, D.FRAME_NUM, D.FRAME_OFFSET, D.SCALE = dataset_dir, frame_num, frame_offset, scale
    D.FIXED_NEAR, D.FIXED_FAR, D.CAMERA_NUM, D.ORIGINAL_SIZE = fixed_near, fixed_far, 0, original_size
    cfg.INPUT = types.SimpleNamespace(SIZE_TEST=list(size_test))
    return cfg
