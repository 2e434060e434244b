"""CPU checks of the class-aware post-processing entry points: the workspace query needs no GPU, and bad arguments come
back as status codes, never as exceptions across the ABI."""


def test_classes_workspace_query_needs_no_gpu():
    import rotate_yolov3_b200 as pkg
    lib = pkg._lib.lib
    assert lib.ryolo_rnms_batched_classes_workspace_bytes(0, 100) > 0
    assert lib.ryolo_rnms_batched_classes_workspace_bytes(3, -1) > 0
    w = lib.ryolo_rnms_batched_classes_workspace_bytes(32, 20000)
    assert w >= 32 * 20032 * 313 * 8               # one mask per image, whatever the number of classes
    assert w >= lib.ryolo_rnms_batched_workspace_bytes(32, 20000)   # plus 64-bit sort keys and the class groups
    assert w < 2 * lib.ryolo_rnms_batched_workspace_bytes(32, 20000)


def test_classes_bad_arguments_return_status():
    import ctypes
    import rotate_yolov3_b200 as pkg
    lib = pkg._lib.lib
    buf = ctypes.c_void_p(256)   # never dereferenced: every call below fails its argument checks first
    sel = lib.ryolo_detect_select_classes
    assert sel(buf, 2, 100, -1, 0.5, 2.0, 10, buf, 10, buf, buf, 1 << 20, None) == -1      # negative class count
    assert sel(buf, 2, 100, 0, 0.5, 2.0, 10, buf, 10, buf, buf, 1 << 20, None) == -1       # no class column
    assert sel(buf, 2, 100, (1 << 24) + 1, 0.5, 2.0, 10, buf, 10, buf, buf, 1 << 20, None) == -1   # ids >= 2^24
    assert sel(buf, 2, 100, 3, 0.5, 2.0, 10, buf, 9, buf, buf, 1 << 20, None) == -1        # cap < limit
    assert sel(buf, 2, 100, 3, -0.5, 2.0, 10, buf, 10, buf, buf, 1 << 20, None) == -1      # conf_thres < 0
    assert b"bad argument" in lib.ryolo_last_error()
    nms = lib.ryolo_rnms_batched_classes
    assert nms(buf, 2, 10, None, 0.5, buf, buf, buf, 1 << 20, None) == -1                  # no device counts
    assert nms(buf, 0, 10, buf, 0.5, buf, buf, buf, 1 << 20, None) == -1                   # no segment
    assert nms(buf, 2, 0, buf, 0.5, buf, buf, buf, 1 << 20, None) == -1                    # cap 0
    assert nms(None, 2, 10, buf, 0.5, buf, buf, buf, 1 << 20, None) == -1                  # no rows
