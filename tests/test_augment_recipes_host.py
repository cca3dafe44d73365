"""CPU: the augmentation recipes' argument checks (TwoViewAugment, get_loader) and the C-ABI binding of the
recipe-taking samplers (no kernel runs)."""
import ctypes
import os
import re

import pytest

from tests.image_folder import loader_kwargs, make_image_folder

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_recipes_and_their_defaults():
    from byol_b200.augment import TwoViewAugment
    ref = TwoViewAugment(224, 1.0, 0)
    assert ref.recipe == "reference" and ref.p_blur == (0.5, 0.5) and ref.p_solarize == (0.0, 0.0)
    assert list(ref._recipe.jitter) == pytest.approx([0.8, 0.8, 0.8, 0.2]) and ref._recipe.bicubic == 0
    byol = TwoViewAugment(224, 1.0, 0, recipe="byol")
    assert byol.p_blur == (1.0, 0.1) and byol.p_solarize == (0.0, 0.2) and byol.ksize == 23
    assert list(byol._recipe.jitter) == pytest.approx([0.4, 0.4, 0.2, 0.1]) and byol._recipe.bicubic == 1
    assert list(byol._recipe.p_blur) == pytest.approx([1.0, 0.1])
    assert list(byol._recipe.p_solarize) == pytest.approx([0.0, 0.2])
    # a scalar means both views; a pair is (view 1, view 2)
    a = TwoViewAugment(64, recipe="byol", p_blur=0.3, p_solarize=(0.5, 1.0))
    assert a.p_blur == (0.3, 0.3) and a.p_solarize == (0.5, 1.0)
    # the existing keyword arguments keep their meaning
    b = TwoViewAugment(image_size=64, seed=3, p_jitter=0.0, p_gray=0.0, p_blur=0.0, blur=False)
    assert b.p == (0.5, 0.0, 0.0) and b.p_blur == (0.0, 0.0) and b.ksize == 0


@pytest.mark.parametrize("kw", [dict(recipe="simclr"), dict(recipe=None), dict(p_blur=1.5), dict(p_blur=(0.1, -0.1)),
                                dict(p_blur=(0.1, 0.2, 0.3)), dict(p_solarize=2.0), dict(p_solarize=(float("nan"), 0.0)),
                                dict(p_flip=-0.5), dict(p_jitter=1.01), dict(p_gray=7)])
def test_two_view_augment_rejects(kw):
    from byol_b200.augment import TwoViewAugment
    with pytest.raises(ValueError):
        TwoViewAugment(64, **kw)


def test_get_loader_augmentation(tmp_path):
    from byol_b200.data import get_loader
    make_image_folder(tmp_path, seed=2)
    ld = get_loader(**loader_kwargs(tmp_path))          # key absent: the reference recipe
    assert ld.augmentation == "reference" and ld.train_loader.augment.recipe == "reference"
    ld = get_loader(**loader_kwargs(tmp_path, augmentation=None))
    assert ld.augmentation == "reference"
    ld = get_loader(**loader_kwargs(tmp_path, augmentation="byol"))
    assert ld.augmentation == "byol" and ld.train_loader.augment.recipe == "byol"
    assert ld.test_loader.augment.recipe == "reference"          # the test split keeps its resize
    with pytest.raises(ValueError):
        get_loader(**loader_kwargs(tmp_path, augmentation="simclr"))


def test_recipe_sampler_bindings():
    from byol_b200 import _lib
    header = open(os.path.join(ROOT, "include", "byol_b200.h")).read()
    for name in ("byol_augment_params_recipe", "byol_augment_params_ragged_recipe"):
        assert name in _lib.EXPORTED_SYMBOLS and re.search(r"\b%s\s*\(" % name, header)
        assert hasattr(ctypes.CDLL(_lib.LIB_PATH), name)
    # the recipe argument is a host pointer to byol_augment_recipe_t; the other arguments follow the scalar entries
    assert _lib._SIGNATURES["byol_augment_params_recipe"][:7] == _lib._SIGNATURES["byol_augment_params"][:7]
    assert _lib._SIGNATURES["byol_augment_params_ragged_recipe"][:8] == _lib._SIGNATURES["byol_augment_params_ragged"][:8]
    # ctypes layout of byol_augment_recipe_t: float jitter[4], p_flip, p_jitter, p_gray, p_blur[2], p_solarize[2],
    # int bicubic
    fields = re.search(r"typedef struct \{(.*?)\} byol_augment_recipe_t;", header, flags=re.S).group(1)
    fields = re.sub(r"/\*.*?\*/", "", fields, flags=re.S)
    names = re.findall(r"(\w+)(?:\[\d\])?\s*[,;]", fields)
    assert names == [f[0] for f in _lib.AugmentRecipe._fields_]
    assert ctypes.sizeof(_lib.AugmentRecipe) == 48 and _lib.AugmentRecipe.bicubic.offset == 44
