"""The public surface of the MLP VAE-engine drop-ins (vae, cvae, bir_vae, aae), without a GPU: for every public class the
public names it adds to nn.Module (models and their modules) or to object (trainers), the signature of each public
callable and the value of each class constant, the public attributes a constructed model and trainer hold, and the
module constants and functions.  The literals are the surface these modules have always had: shared plumbing behind
them must neither add a name to one drop-in nor take one away."""
import inspect

import pytest
import torch
import torch.nn as nn

import aae
import bir_vae
import cvae
import vae

TRAINER = "(model, train_iter, val_iter, test_iter, viz=False)"
TRAIN = "(self, num_epochs, lr=0.001, weight_decay=1e-05)"
COMMON = {"(class)": TRAINER, "device_noise": "True", "evaluate": "(self, iterator)", "load_model": "(self, loadpath)",
          "save_model": "(self, savepath)", "viz_loss": "(self)", "compute_batch": "(self, batch)", "train": TRAIN,
          "reconstruct_images": "(self, images, epoch, save=True)",
          "sample_images": "(self, epoch=-100, num_images=36, save=True)"}
LATENT_VIZ = {"explore_latent_space": "(self, num_epochs=3)", "make_all": "(self)", "sample_interpolated_images": "(self)"}
KL = {"kl_divergence": "(self, mu, log_var)"}

CLASSES = {
    vae: {
        "Encoder": {"(class)": "(image_size, hidden_dim, z_dim)", "forward": "(self, x)"},
        "Decoder": {"(class)": "(z_dim, hidden_dim, image_size)", "forward": "(self, z)"},
        "VAE": {"(class)": "(image_size=784, hidden_dim=400, z_dim=20)", "forward": "(self, x)",
                "reparameterize": "(self, mu, log_var)"},
        "VAETrainer": {**COMMON, **LATENT_VIZ, **KL},
    },
    cvae: {
        "Encoder": {"(class)": "(image_size, hidden_dim, z_dim, num_classes)", "forward": "(self, x, y)"},
        "Decoder": {"(class)": "(z_dim, hidden_dim, image_size, num_classes)", "forward": "(self, z, y)"},
        "CVAE": {"(class)": "(image_size=784, hidden_dim=400, z_dim=20, num_classes=10)", "forward": "(self, x, y)",
                 "reparameterize": "(self, mu, log_var)"},
        "CVAETrainer": {**COMMON, **KL, "reconstruct_images": "(self, images, labels, epoch, save=True)",
                        "sample_images": "(self, epoch=-100, num_images=36, save=True, labels=None)"},
    },
    bir_vae: {
        "Encoder": {"(class)": "(image_size, hidden_dim, z_dim)", "forward": "(self, x)"},
        "Decoder": {"(class)": "(z_dim, hidden_dim, image_size)", "forward": "(self, z)"},
        "BIRVAE": {"(class)": "(image_size=784, hidden_dim=400, z_dim=20, I=13.3)", "forward": "(self, x)",
                   "reparameterize": "(self, mu)"},
        "BIRVAETrainer": {**COMMON, **LATENT_VIZ, "compute_batch": "(self, batch, LAMBDA=1000.0)",
                          "compute_kernel": "(self, x, y)", "maximum_mean_discrepancy": "(self, z)"},
    },
    aae: {
        "Encoder": {"(class)": "(image_size, hidden_dim, z_dim)", "forward": "(self, x)"},
        "Decoder": {"(class)": "(z_dim, hidden_dim, image_size)", "forward": "(self, z)"},
        "Discriminator": {"(class)": "(z_dim, hidden_dim, output_dim=1)", "forward": "(self, z)"},
        "AAE": {"(class)": "(image_size=784, hidden_dim=400, z_dim=20)", "forward": "(self, x)"},
        "AAETrainer": {**COMMON, "train": "(self, num_epochs, lr=0.001, D_lr=0.0002, G_lr=0.0002, weight_decay=1e-05)",
                       "train_D": "(self, images)", "train_G": "(self, images)"},
    },
}

CONSTANTS = {
    vae: {},
    cvae: {"MAX_LATENT_ROW": 63,
           "VAE_EPOCH_LINE": "Epoch[%d/%d], Total Loss: %.4f, Reconst Loss: %.4f, KL Div: %.7f, Val Loss: %.4f"},
    bir_vae: {"EPOCH_LINE": "Epoch[%d/%d], Total Loss: %.4f, MSE Loss: %.4f, MMD Loss: %.4f, Val Loss: %.4f"},
    aae: {"EPOCH_LINE": "Epoch[%d/%d], Recon Loss: %.4f, D Loss: %.4f, G Loss: %.4f, Val Loss: %.4f"},
}
FUNCTIONS = {vae: {}, cvae: {}, bir_vae: {},
             aae: {"has_custom_step": "(tr)", "reference_loop": "(tr, num_epochs, lr, D_lr, G_lr, weight_decay)"}}

TRAINER_ATTRS = ["best_val_loss", "debugging_image", "model", "name", "num_epochs", "recon_loss", "test_iter",
                 "train_iter", "val_iter", "viz"]
INSTANCES = {   # (model class, trainer class, the model's public attributes, the trainer's beyond TRAINER_ATTRS)
    vae: ("VAE", "VAETrainer", ["hidden_dim", "image_size", "shape", "z_dim"], ["kl_loss"]),
    cvae: ("CVAE", "CVAETrainer", ["hidden_dim", "image_size", "num_classes", "shape", "z_dim"],
           ["debugging_labels", "kl_loss"]),
    bir_vae: ("BIRVAE", "BIRVAETrainer", ["I", "hidden_dim", "image_size", "set_var", "shape", "z_dim"], ["mmd_loss"]),
    aae: ("AAE", "AAETrainer", ["hidden_dim", "image_size", "shape", "z_dim"], ["Dlosses", "Glosses"]),
}


def _surface(cls):
    """{public name cls adds to nn.Module (or object): its signature, or the repr of a constant} and cls's own signature"""
    module = issubclass(cls, nn.Module)
    names = sorted(n for n in set(dir(cls)) - set(dir(nn.Module if module else object)) if not n.startswith("_"))
    out = {"(class)": str(inspect.signature(cls))}
    for n in names + (["forward"] if module else []):
        a = getattr(cls, n)
        out[n] = str(inspect.signature(a)) if callable(a) else repr(a)
    return out


def _module_names(mod):
    """the public classes, functions and constants mod defines itself (not the names it imports)"""
    classes, functions, constants = set(), set(), set()
    for n, v in vars(mod).items():
        if n.startswith("_"):
            continue
        if isinstance(v, type) and v.__module__ == mod.__name__:
            classes.add(n)
        elif inspect.isfunction(v) and v.__module__ == mod.__name__:
            functions.add(n)
        elif isinstance(v, (int, float, str, bool, tuple)):
            constants.add(n)
    return classes, functions, constants


@pytest.mark.parametrize("mod", list(CLASSES), ids=lambda m: m.__name__)
def test_public_classes_names_and_signatures(mod):
    classes, functions, constants = _module_names(mod)
    assert classes == set(CLASSES[mod])
    for name, expected in CLASSES[mod].items():
        assert _surface(getattr(mod, name)) == expected, name
    assert functions == set(FUNCTIONS[mod])
    for name, sig in FUNCTIONS[mod].items():
        assert str(inspect.signature(getattr(mod, name))) == sig
    assert constants == set(CONSTANTS[mod])
    for name, value in CONSTANTS[mod].items():
        assert getattr(mod, name) == value


def test_what_a_drop_in_does_not_have():
    for name in ("kl_divergence", "sample_interpolated_images", "explore_latent_space", "make_all",
                 "maximum_mean_discrepancy"):
        assert not hasattr(aae.AAETrainer, name), name
    for name in ("explore_latent_space", "sample_interpolated_images", "make_all", "maximum_mean_discrepancy"):
        assert not hasattr(cvae.CVAETrainer, name), name
    assert not hasattr(bir_vae.BIRVAETrainer, "kl_divergence")
    assert not hasattr(vae.VAETrainer, "maximum_mean_discrepancy")


@pytest.mark.parametrize("mod", list(INSTANCES), ids=lambda m: m.__name__)
def test_public_attributes_of_a_model_and_its_trainer(mod):
    model_name, trainer_name, model_attrs, trainer_attrs = INSTANCES[mod]
    x = (torch.rand(8, 1, 28, 28) < 0.5).float()
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(x, torch.zeros(8, dtype=torch.long)), batch_size=4)
    model = getattr(mod, model_name)(784, 32, 4)
    tr = getattr(mod, trainer_name)(model, loader, loader, loader)
    assert sorted(k for k in vars(model) if not k.startswith("_") and k != "training") == model_attrs
    assert sorted(k for k in vars(tr) if not k.startswith("_")) == sorted(TRAINER_ATTRS + trainer_attrs)
    assert tr.name == model_name and tr.recon_loss == [] and tr.num_epochs == 0 and tr.best_val_loss == 1e10
