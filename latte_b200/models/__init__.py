"""Drop-in for the reference's `models` package factory (Vchitect/Latte models/__init__.py:31-51).

`sample/sample.py:56`, `sample/sample_ddp.py:88` and `train.py:90` call `get_models(args)`; putting this
package ahead of the reference's on sys.path (see INTEGRATION.md) swaps the denoiser and nothing else."""
from latte_b200.latte import Latte, Latte_models  # noqa: F401  (absolute: also importable as top-level `models` via a symlink)
from latte_b200.latte_img import LatteIMG, LatteIMG_models  # noqa: F401


def get_models(args):
    name = args.model
    if "LatteIMG" in name:
        # models/__init__.py:32-38 (train_with_img.py).  The conditioning is checked first: extras=78 (the legacy CLIP text
        # projection) is not built, and neither is an argument set that names no conditioning at all.
        extras = getattr(args, "extras", None)
        if extras not in (1, 2):
            raise NotImplementedError(f"{name} with extras={extras!r}: LatteIMG is built for extras=2 (class labels, per-image "
                                      "labels in training) and extras=1 (timestep only)")
        return LatteIMG_models[name](input_size=args.latent_size, num_classes=args.num_classes,
                                     num_frames=args.num_frames, learn_sigma=args.learn_sigma, extras=args.extras)
    if "LatteT2V" in name:
        # models/__init__.py:40-41
        from latte_b200.latte_t2v import LatteT2V
        return LatteT2V.from_pretrained(args.pretrained_model_path, subfolder="transformer", video_length=args.video_length)
    if "Latte" in name:
        # same keyword set as the reference factory (models/__init__.py:42-49)
        return Latte_models[name](input_size=args.latent_size, num_classes=args.num_classes,
                                  num_frames=args.num_frames, learn_sigma=args.learn_sigma, extras=args.extras)
    raise ValueError(f"{name} Model Not Supported!")
