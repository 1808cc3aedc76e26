"""CPU oracle for the Luminoth Faster R-CNN / SSD inference hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``luminoth_b200/`` imports this
package; only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline``
/ ``--impl reference`` legs of ``bench.py`` may.  It is the checker, never the
product: the product path is the sm_90a CUDA library and fails loudly when
that library is missing.

What it restates (reference = tryolabs/luminoth @ 9109d8b, paths relative to
``luminoth/``):

* ``tf_ops``      TensorFlow-1.x op semantics the reference delegates to
                  (conv2d SAME/VALID, slim batch_norm, max_pool,
                  crop_and_resize, non_max_suppression, top_k, softmax,
                  resize_images, l2_normalize).  TF is a third-party,
                  un-vendored dependency (``setup.py:107``, unpinned >=1.5);
                  the semantics are restated from its published kernels.
* ``bbox``        ``utils/bbox_transform_tf.py:4-126``, ``utils/bbox_transform.py:105-122``
* ``anchors``     ``utils/anchors.py:4-52``, ``models/fasterrcnn/fasterrcnn.py:261-308``,
                  ``models/ssd/utils.py:5-145``
* ``resnet``      slim ``resnet_v1_{50,101}`` trunk to ``block3`` and the
                  R101 ``block4`` tail (``models/base/base_network.py:69-177``,
                  ``models/base/truncated_base_network.py:8-95``)
* ``vgg``         ``models/base/truncated_vgg.py:60-121`` and the SSD extra
                  layers (``models/ssd/feature_extractor.py:27-132``)
* ``fasterrcnn``  ``models/fasterrcnn/{fasterrcnn,rpn,rpn_proposal,roi_pool,rcnn,rcnn_proposal}.py``
* ``ssd``         ``models/ssd/{ssd,proposal}.py``
* ``predict``     ``utils/predicting.py:109-148`` + ``utils/image.py:38-147``

Parity pinning: the reference cannot be imported here (TensorFlow 1.x and
dm-sonnet are not installable: no cp312 wheels, no network), so the oracle is
pinned against every known-answer test the reference holds for this path
(ported in ``tests/test_oracle_reference_goldens.py`` with file:line cites).
The backbone / head convolution numerics and all of SSD have no such vectors
in the reference: for those the header says it plainly -- **parity unpinned**
(cross-checked only against ``torch.nn.functional`` and an fp64 run of
this same restatement).
"""
