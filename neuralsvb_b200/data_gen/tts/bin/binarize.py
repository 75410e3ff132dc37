"""The reference's binarize entry point (data_gen/tts/bin/binarize.py):

    python -m neuralsvb_b200.data_gen.tts.bin.binarize --config egs/svb_binarize_synthetic.yaml [--hparams "k=v,..."]

runs ``hparams['binarizer_cls']().process()``.  A class path of the reference's layout (``data_gen.singing.binarize_para...``) is
looked up in this package."""
import importlib

from neuralsvb_b200.utils.hparams import hparams, set_hparams


def binarizer_class(path):
    pkg, _, cls_name = path.rpartition('.')
    if pkg.startswith('data_gen.'):
        pkg = 'neuralsvb_b200.' + pkg
    return getattr(importlib.import_module(pkg), cls_name)


def binarize():
    binarizer_cls = binarizer_class(hparams.get('binarizer_cls', 'neuralsvb_b200.data_gen.singing.binarize_para.PopBuTFyENSpkEMBinarizer'))
    print("| Binarizer: ", binarizer_cls)
    binarizer_cls().process()


if __name__ == '__main__':
    set_hparams()
    binarize()
