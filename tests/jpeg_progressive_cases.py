"""Progressive JPEG files (tests/golden/make_golden_jpeg_progressive.py builds them and writes tests/golden/jpeg_progressive.npz
with cv2 and Pillow).  The npz holds "jpg_<name>" and, of cv2.imdecode(bytes, IMREAD_COLOR), either "none_<name>" or the frame
as jpeg_cases does ("shape_", "sha_" and, up to jpeg_cases.FULL_BYTES, "bgr_"), so jpeg_cases.equals_golden compares against it.

The families:
- cv2_*:    cv2.imencode(IMWRITE_JPEG_PROGRESSIVE) of every sampling of jpeg_cases.SAMPLINGS at q1/50/95/100, its size ladder,
            restart intervals 1 and 7, EXIF 6 and 8 in both byte orders, a 1080p 4:2:0 frame;
- pil_*:    Pillow's progressive=True at subsampling 0/1/2 x q5/50/95, optimize, grey;
- tx_*:     the reference's two photos re-coded losslessly as progressive files (their own coefficients and tables), with cv2's
            script (tx_cv2_*) and a seeded script with AC approximation chains (tx_seeded_*): cv2 decodes both to
            frames_modelzoo.npz's frames;
- script_*: the generator's encoder, seeded complete scripts over three coefficient sets (37x53 4:2:0, 31x33 4:4:4 at q1, 37x53
            grey): DC interleaved over all, 2 + 1 or one per component, DC chains from Al up to 13, random bands, 1-wide bands
            and band 63 alone; script_ac_* add AC approximation chains (AC refinement from Al up to 13 over random, narrow
            and 1-wide bands); script_<set>_flat is the same coefficients in one scan per component group;
- enc_*:    DRI changed between scans, restart intervals not dividing a block row, EOB runs past their segment's end, EOB14 over
            many rows, extreme DC and AC at Al 13, ZRL in AC refinement, and cv2 files rewritten: DQT redefined after a
            component's first scan, a DC refinement naming undefined tables, refinement symbols of size 2 (enc_base is the
            file they were rewritten from);
- bad_* / bogus_*: refused (REFUSED: code and a substring of the reason);
- cut_*, corrupt_*, rst_*: damaged scans (DAMAGED), the only accepted files allowed a flag.

Every accepted file without a flag decodes to cv2's bytes."""

CASES = []
_SAMPLINGS = ("444", "422", "420", "440", "411", "grey")
for _s in _SAMPLINGS:
    CASES += ["cv2_q%d_%s" % (q, _s) for q in (1, 50, 95, 100)]
    CASES += ["cv2_size%dx%d_%s" % (h, w, _s) for (h, w) in ((1, 1), (1, 17), (17, 1), (8, 8), (15, 9), (16, 16), (31, 33),
                                                              (37, 53), (333, 500))]
    CASES += ["cv2_rst%d_%s" % (r, _s) for r in (1, 7)]
CASES += ["cv2_exif%d_%s" % (o, b) for o in (6, 8) for b in ("II", "MM")] + ["cv2_fullhd_420"]
CASES += ["pil_sub%d_q%d" % (s, q) for s in (0, 1, 2) for q in (5, 50, 95)] + ["pil_optimize", "pil_grey"]
PHOTOS = ("000004", "000139")
CASES += ["tx_%s_%s" % (k, s) for s in PHOTOS for k in ("cv2", "seeded")]
for _set in ("420", "444", "grey"):
    CASES += ["script_%s_%d" % (_set, k) for k in range(6)] + ["script_ac_%s_%d" % (_set, k) for k in range(6)]
    CASES += ["script_%s_flat" % _set]
CASES += ["script_grey_wide"]
CASES += ["enc_dri_between_scans", "enc_rst_not_row", "enc_eob_past_segment", "enc_eob14_rows", "enc_dc_al13", "enc_base",
          "enc_dqt_after_first_scan", "enc_dc_refine_undefined_tables", "enc_refine_size2", "enc_ac_al13", "enc_zrl_refine"]

EINVAL, EUNSUPPORTED = -1, -3
REFUSED = {"bad_first_%d_scans" % k: (EUNSUPPORTED, "incomplete progressive") for k in range(1, 10)}
REFUSED.update({
    "bad_component_never_scanned": (EUNSUPPORTED, "component 1 coefficient 0 is never sent"),
    "bad_dc_se1": (EINVAL, "bad progressive scan 0: a DC scan with Se = 1"),
    "bad_ac_ss_after_se": (EINVAL, "bad progressive scan 1: coefficients 6..5"),
    "bad_ac_se64": (EINVAL, "bad progressive scan 1: coefficients 1..64"),
    "bad_ac_two_components": (EINVAL, "bad progressive scan 1: an AC scan of 2 components"),
    "bad_ah_al": (EINVAL, "bad progressive scan 5: Ah 2 with Al 0"),
    "bad_al14": (EINVAL, "bad progressive scan 0: Al 14"),
    "bogus_ac_before_dc": (EUNSUPPORTED, "bogus progressive scan 0: AC of component 0 before its DC"),
    "bogus_ah": (EUNSUPPORTED, "bogus progressive scan 5: component 0 coefficient 1 has Ah 3, 2 expected"),
    "bad_too_many_scans": (EUNSUPPORTED, "more than 128 scans"),
    "bad_sof10": (EUNSUPPORTED, "arithmetic-coded progressive (SOF10)"),
    "bad_dc_components_out_of_order": (EUNSUPPORTED, "progressive scan 0: components not in frame order"),
})
CASES += list(REFUSED)

DAMAGED = ["cut_first_scan", "cut_refinement", "cut_between_scans", "cut_before_eoi", "cut_eoi_d9"]
DAMAGED += ["corrupt_refinement_%d" % k for k in range(3)] + ["corrupt_run_past_band", "rst_renumbered_in_refinement"]
CASES += DAMAGED
