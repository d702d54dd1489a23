"""
genomad_b200 -- H100-native (sm_90a) implementation of geNomad's ``nn-classification`` hot path.

Public surface (mirrors the reference's for this path only):
  genomad_b200.nn_classification.main(input_path, output_path, single_window, batch_size, restart,
                                      threads, verbose, cleanup)     <- genomad.nn_classification.main
  genomad_b200.cli.nn_classification                                 <- `genomad nn-classification`
  genomad_b200.engine.Classifier                                     <- create_classifier() + predict()
"""
__version__ = "0.2.0"
