"""JPEG files cv2.imencode did not write (tests/golden/make_golden_jpeg_foreign.py builds them and writes
tests/golden/jpeg_foreign.npz with cv2 and Pillow).  The npz holds "jpg_<name>" (the file's bytes) and, of cv2.imdecode(bytes,
IMREAD_COLOR), either "none_<name>" (it returned None) or the frame as jpeg_cases does: "shape_<name>", "sha_<name>" and, up to
jpeg_cases.FULL_BYTES, "bgr_<name>" (so jpeg_cases.equals_golden compares against either).

The families:
- pil_*:     Pillow's encoder (subsampling 0/1/2 at q5/50/95, its qtables, restart rows / blocks, optimize, smooth, ICC + COM, grey);
- enc_*:     the generator's own encoder (a table per component, 16-bit DQT under SOF0 and SOF1, restart intervals that do not
             divide the MCU row);
- hdr_*:     cv2 files with rewritten headers (fill bytes, table layout, redefined tables, component ids, JFIF / Adobe, RGB ids,
             bytes after EOI, no EOI);
- exif_*:    EXIF APP1 variants in both byte orders (entry types, counts, values, IFD placement, truncation, two APP1s, XMP first,
             APP1 after DQT);
- huff_*, ac_*, extreme_*: hand-built Huffman tables and symbol streams (9-, 10-, 15- and 16-bit codes, one-symbol tables, AC
             sizes 11-15, ZRL runs ending at or past coefficient 63, coefficients whose dequantised values and IDCT passes leave
             int16, DC predictors walking outside int16);
- corrupt_*, rst_*, cut_*: damaged scans (seeded byte changes, stray markers and FF bytes inside the scan, RSTn dropped /
             duplicated / renumbered / extra, truncation).

Every file the decoder accepts must decode to cv2's bytes unless the decode flags it; DAMAGED and the files cv2 cannot decode are
the only cases allowed a flag.
REFUSED: the files the parser refuses, name -> (parse code, a substring of the reason)."""

CASES = []
CASES += ["pil_sub%d_q%d" % (s, q) for s in (0, 1, 2) for q in (5, 50, 95)]
CASES += ["pil_qtables3", "pil_qtables2_420", "pil_qtables1", "pil_rst_rows", "pil_rst_blocks", "pil_optimize", "pil_smooth",
          "pil_icc_com", "pil_grey"]
CASES += ["enc_qt_percomp", "enc_dqt16_le255", "enc_dqt16_1023_sof1", "enc_rst3_of7", "enc_rst5_of7", "enc_rst9_of7"]
CASES += ["hdr_plain", "hdr_fill", "hdr_fill_rst", "hdr_tables_combined", "hdr_tables_split", "hdr_tables_after_sof",
          "hdr_tables_redefined", "hdr_ids_012", "hdr_ids_arbitrary", "hdr_no_jfif", "hdr_adobe1", "hdr_adobe1_rgb_ids",
          "hdr_rgb_ids_jfif", "hdr_rgb_ids_short_jfif", "hdr_rgb_ids_no_jfif", "hdr_garbage_after_eoi", "hdr_no_eoi"]
for _o in ("II", "MM"):
    CASES += ["exif_%s_%s_6" % (_o, t) for t in ("byte", "short", "long", "undef", "slong")]
    CASES += ["exif_%s_long_0x60000" % _o, "exif_%s_count0" % _o] + ["exif_%s_value%d" % (_o, v) for v in (0, 9, 0x0106)]
    CASES += ["exif_%s_%s" % (_o, k) for k in ("ifd_at_20", "third_entry", "truncated_ifd", "truncated_value", "truncated_entry_10",
                                               "truncated_entry_11", "one_entry_truncated", "count_past_end", "two_app1",
                                               "xmp_first", "after_dqt")]
CASES += ["huff_9bit", "huff_10bit", "huff_9_10bit", "huff_8_9_10bit", "huff_16bit", "huff_15_16bit", "huff_one_symbol",
          "huff_one_ac_symbol", "ac_size_11_15", "ac_zrl_runs_to_63"]
CASES += ["extreme_grey_%d" % s for s in range(6)] + ["extreme_420_%d" % s for s in range(2)] + ["extreme_dc_only", "extreme_dc_walk"]
CASES += ["corrupt_bytes_%d" % s for s in range(8)] + ["corrupt_marker_%s" % m for m in ("ff01", "ffc4", "ffe0", "ffd9", "ffd0")]
CASES += ["corrupt_ff_written_%d" % s for s in range(3)]
CASES += ["rst_dropped_3", "rst_dropped_last", "rst_duplicated_3"] + ["rst_renumbered_5_plus%d" % d for d in range(1, 8)]
CASES += ["rst_extra_past_last", "rst_extra_empty_past_last"]
CASES += ["cut_scan_10", "cut_scan_50", "cut_scan_97", "cut_inside_ff00", "cut_after_ff00", "cut_before_eoi_ff"]

DAMAGED = [c for c in CASES if c.split("_")[0] in ("corrupt", "rst", "cut")]

REFUSED = {
    "hdr_rgb_ids_short_jfif": (-3, "RGB-coded (component ids R, G, B)"),
    "hdr_rgb_ids_no_jfif": (-3, "RGB-coded (component ids R, G, B)"),
}
