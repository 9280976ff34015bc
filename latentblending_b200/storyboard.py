"""Storyboard JSON + the multi-transition driver (SURVEY.md section 8f "next #4").

The reference stores a movie as a JSON list (gradio_ui.py:168-191 ``write_json`` / ``add_image_to_video``):
element 0 = settings ``{"settings": "sdxl", "width": W, "height": H, "num_inference_steps": N}``, then one
element per key frame ``{"iteration": i, "seed": s, "prompt": p, "negative_prompt": n, "preview_image": ...}``.
``example_multi_trans_json.py:26-74`` replays it: dimensions and step count from the settings, then for every
consecutive prompt pair one ``run_transition`` -- the first with both prompts set, the later ones after
``swap_forward()`` with ``recycle_img1=True`` -- followed by ``write_movie_transition`` per part.
This module is that file format and loop for this backend's BlendingEngine (same call order, including the
reference's negative-prompt indexing: entry 0's negative prompt for the first transition, entry i+1's afterwards).
A key frame may also start from an image (BlendingEngine.set_init_image1/2): ``"init_image"``, a path relative to the
JSON file, and ``"strength"`` (default 0.3).
"""
import json
import os


def load_storyboard(fp_json):
    """-> (settings dict, prompts, negative_prompts, seeds) like example_multi_trans_json.py:26-47."""
    with open(fp_json, "r") as f:
        data = json.load(f)
    if not isinstance(data, list) or len(data) < 3:
        raise ValueError("a storyboard needs a settings element and at least two key frames")
    settings = data[0]
    for k in ("width", "height", "num_inference_steps"):
        if k not in settings:
            raise ValueError(f"storyboard settings lack '{k}'")
    prompts = [item["prompt"] for item in data[1:]]
    negative_prompts = [item.get("negative_prompt", "") for item in data[1:]]
    seeds = [int(item["seed"]) for item in data[1:]]
    return settings, prompts, negative_prompts, seeds


DEFAULT_STRENGTH = 0.3


def load_init_images(fp_json):
    """-> one (init image path or None, strength) per key frame: ``init_image`` resolved against the JSON file's
    directory, ``strength`` defaulting to 0.3."""
    with open(fp_json, "r") as f:
        data = json.load(f)
    base = os.path.dirname(os.path.abspath(fp_json))
    out = []
    for item in data[1:]:
        p = item.get("init_image")
        out.append((None if p is None else os.path.normpath(os.path.join(base, p)),
                    float(item.get("strength", DEFAULT_STRENGTH))))
    return out


def write_storyboard(fp_json, be, entries, settings_name="sdxl"):
    """gradio_ui.py:168-174: ``entries`` = dicts with prompt / negative_prompt / seed (iteration is filled in), and
    optionally init_image (a path, written as given: relative paths are relative to the JSON file) and strength."""
    data = [{"settings": settings_name, "width": be.dh.width_img, "height": be.dh.height_img,
             "num_inference_steps": be.dh.num_inference_steps}]
    for i, e in enumerate(entries):
        data.append({"iteration": i, "seed": int(e["seed"]), "prompt": e["prompt"],
                     "negative_prompt": e.get("negative_prompt", ""), "preview_image": e.get("preview_image")})
        if e.get("init_image") is not None:
            data[-1]["init_image"] = e["init_image"]
            data[-1]["strength"] = float(e.get("strength", DEFAULT_STRENGTH))
    with open(fp_json, "w") as f:
        json.dump(data, f, indent=4)
    return data


def _open_image(img):
    if isinstance(img, (str, os.PathLike)):
        from PIL import Image
        with Image.open(img) as im:
            return im.convert("RGB")
    return img


def run_multi_transition(be, prompts, seeds, negative_prompts=None, on_transition=None, init_images=None):
    """The multi-transition loop (example_multi_trans.py:38-62 / example_multi_trans_json.py:49-74).
    Yields (i, frames) per transition; ``on_transition(i, be)`` runs after each (e.g. write_movie_transition).
    ``init_images``: None (every key frame text-only, without touching the engine's image keyframes) or one
    (image | path | None, strength) per key frame, set with set_init_image1/2 (swap_forward carries key frame i+1's
    image to the next transition)."""
    assert len(prompts) >= 2 and len(seeds) == len(prompts)
    assert init_images is None or len(init_images) == len(prompts)
    for i in range(len(prompts) - 1):
        if i == 0:
            be.set_prompt1(prompts[i])
            if negative_prompts is not None:
                be.set_negative_prompt(negative_prompts[i])
            be.set_prompt2(prompts[i + 1])
            if init_images is not None:
                img, strength = init_images[0]
                be.set_init_image1(_open_image(img), strength)
            recycle_img1 = False
        else:
            be.swap_forward()
            if negative_prompts is not None:
                be.set_negative_prompt(negative_prompts[i + 1])
            be.set_prompt2(prompts[i + 1])
            recycle_img1 = True
        if init_images is not None:
            img, strength = init_images[i + 1]
            be.set_init_image2(_open_image(img), strength)
        frames = be.run_transition(recycle_img1=recycle_img1, fixed_seeds=list(seeds[i:i + 2]))
        if on_transition is not None:
            on_transition(i, be)
        yield i, frames


def run_storyboard(be, fp_json, dp_out=None, duration_single_trans=10, fps=30, init_images=None):
    """Replay a storyboard JSON: set dimensions / steps from its settings, run every transition and -- when ``dp_out``
    is given -- write one movie part per transition (``tmp_part_000.mp4`` ..., example_multi_trans_json.py:66-71).
    Returns the list of part paths (or of frame lists when no output directory is given).  Concatenating the parts is
    the reference's lunar_tools.concatenate_movies (ffmpeg), outside this backend.
    ``init_images``: as run_multi_transition's; None takes the storyboard's own ``init_image`` / ``strength`` fields,
    and a storyboard without any runs text-only as before."""
    settings, prompts, negative_prompts, seeds = load_storyboard(fp_json)
    if init_images is None:
        init_images = load_init_images(fp_json)
        if all(p is None for p, _ in init_images):
            init_images = None
    be.set_dimensions((settings["width"], settings["height"]))
    be.set_num_inference_steps(settings["num_inference_steps"])
    out = []

    def after(i, engine):
        if dp_out is not None:
            os.makedirs(dp_out, exist_ok=True)
            fp = os.path.join(dp_out, f"tmp_part_{str(i).zfill(3)}.mp4")
            engine.write_movie_transition(fp, duration_single_trans, fps=fps)
            out.append(fp)

    for i, frames in run_multi_transition(be, prompts, seeds, negative_prompts, on_transition=after,
                                          init_images=init_images):
        if dp_out is None:
            out.append(frames)
    return out
