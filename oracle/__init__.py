"""CPU oracle for the RetinaFace mnet25 detect path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is part of the product: only
``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference``
legs of ``bench.py`` may import, link or execute it, and only as the checker or the timed
CPU baseline -- never as the path being measured or shipped.  The product
(``retinaface_b200`` + ``librf_b200.so``) has no CPU fallback and fails loudly without its
CUDA library.

Pieces (each function cites the reference file:line it restates):

* ``caffemodel.py``   -- protobuf-wire reader for the reference's ``*.caffemodel`` files.
* ``topology.py``     -- the mnet25 / mnet-deconv-0517 layer graph (restated from
                         ``model/mnet-deconv-0517.prototxt``) + a prototxt writer so that
                         ``cv2.dnn`` can execute it where /root/reference is absent.
* ``mnet_numpy.py``   -- FP32 numpy restatement of the Caffe forward pass (9 head blobs).
* ``mnet_int8.py``    -- integer oracle of the INT8 path: the exact quantisation scheme of RF_PREC_INT8 on the
                         reference's calibration-table scales (TensorRT's own INT8 kernels are closed source).
* ``calibrator_ref.py`` -- numpy restatement of the entropy-calibration threshold search of rf_calibrate_int8.
* ``inputs.py``       -- the reference's OpenCV letter-box branch + the seeded synthetic inputs of SURVEY 8d.
* ``letterbox.py``    -- numpy restatement of the letter-box kernels' own definition (both resize branches, the 2x
                         area rule, orientations), checked against cv2 and held against the kernels.
* ``postproc.c``      -- plain-C restatement of anchors / decode / clip / NMS
                         (``retinaface/RetinaFace.cpp:9-199,347-492,661-726``).
* ``postproc.py``     -- ctypes loader for the C restatement and for ``oracle/_ref``.
* ``build_ref.sh``    -- compiles the reference's own ``RetinaFace.cpp`` (unmodified, from
                         where it lies in /root/reference) against stub headers in
                         ``oracle/shim`` into ``oracle/_ref/libref_postproc.so``.

Pinning status: the reference has NO tests / golden vectors (SURVEY.md section 4), so the
oracle is pinned against *outputs of the reference itself run here*: the post-process
restatement against ``oracle/_ref`` (the reference's own compiled code) and the forward
restatement against ``cv2.dnn`` executing the reference's own prototxt + caffemodel
(fixtures + generating script under ``tests/golden``).
"""
