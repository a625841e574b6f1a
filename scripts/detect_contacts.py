#!/usr/bin/env python
"""Drop-in for `python contact_learning/test.py --data D --out O --weights-path W --full-video --save-contacts
--real-data` (reference scripts/run_detect_contacts.py:51-58): writes O/contact_results/<video>/foot_contacts.npy
(int64, F x 4, columns L heel, L toe, R heel, R toe).  With `--copy-into-data` it also performs
run_detect_contacts.py:65-69 (copy into each video directory).  Flags the reference ignores for saved labels
(--classify-thresh, test.py:88) are accepted and ignored too."""
import argparse
import os
import shutil
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--data", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--weights-path", "--weights", dest="weights", required=True)
    ap.add_argument("--full-video", action="store_true")
    ap.add_argument("--save-contacts", action="store_true")
    ap.add_argument("--real-data", action="store_true")
    ap.add_argument("--viz", action="store_true")
    ap.add_argument("--classify-thresh", type=float, default=0.5)
    ap.add_argument("--copy-into-data", action="store_true")
    ap.add_argument("--precision", choices=["fp32", "tf32x3"], default="fp32",
                    help="fp32: labels match the reference's fp32 forward; tf32x3: the large layers on the tensor core "
                         "with split TF32 operands")
    args = ap.parse_args(argv)
    import chd
    sd = chd.contact.load_weights(args.weights)
    written = chd.contact.detect_contacts(args.data, args.out, sd, precision=args.precision)
    for w in written:
        print("wrote", w)
        if args.copy_into_data:
            vid = os.path.basename(os.path.dirname(w))
            shutil.copyfile(w, os.path.join(args.data, vid, "foot_contacts.npy"))


if __name__ == "__main__":
    main()
