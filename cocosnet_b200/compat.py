"""Drop-in aliasing for code written against the reference's module paths
(`models.pix2pix_model`, `models.networks`, `trainers.pix2pix_trainer`,
`options.train_options`, `options.test_options`, `util.util`): after
`cocosnet_b200.compat.install()` those imports resolve to this package, so the
reference's own train.py / test.py drive the native path unmodified apart from
their data loader (INTEGRATION.md)."""
import sys
import types


def install():
    from . import nets, options, pix2pix_model, trainer, util

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    mod("models", create_model=lambda opt: pix2pix_model.Pix2PixModel(opt),
        get_option_setter=lambda name: pix2pix_model.Pix2PixModel.modify_commandline_options)
    sys.modules["models.pix2pix_model"] = pix2pix_model
    sys.modules["models.networks"] = nets
    sys.modules["models.networks.correspondence"] = nets.correspondence
    sys.modules["models.networks.generator"] = nets.generator
    sys.modules["models.networks.discriminator"] = nets.discriminator
    mod("trainers")
    sys.modules["trainers.pix2pix_trainer"] = trainer
    mod("options")
    mod("options.train_options", TrainOptions=options.TrainOptions)
    mod("options.test_options", TestOptions=options.TestOptions)
    mod("options.base_options", BaseOptions=options.BaseOptions)
    mod("util")
    sys.modules["util.util"] = util
