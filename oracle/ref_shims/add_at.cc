/* add_at.cc -- TEST INFRASTRUCTURE: `audiowmark add` of the UNMODIFIED reference with a stream offset.
 *
 * The reference reaches add_stream_watermark with zero_frames != 0 only through hls-add (src/hls.cc:244-279, zero_frames =
 * start_pos - prev_size), which needs ffmpeg for the MPEG-TS side.  This driver links the reference's own object files (compiled
 * where they lie by oracle/Makefile.ref, everything except audiowmark.o) and calls add_stream_watermark (src/wmadd.cc:448-618)
 * on a WAV file with a given zero_frames, writing the result as 16 bit PCM, as `audiowmark add` does for a 16 bit input.  The
 * "SNR" and "Data Blocks" lines go to stderr as the reference prints them.  All arithmetic is the reference's; only this argument
 * parsing is ours.
 *
 *   add_at [--snr] [--test-no-limiter] in.wav out.wav <payload hex> <zero_frames>
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <memory>
#include <string>

#include "wmcommon.hh"
#include "audiostream.hh"
#include "random.hh"

int
main (int argc, char **argv)
{
  int a = 1;
  for (; a < argc && !strncmp (argv[a], "--", 2); a++)
    {
      if (!strcmp (argv[a], "--snr"))
        Params::snr = true;
      else if (!strcmp (argv[a], "--test-no-limiter"))
        Params::test_no_limiter = true;
      else
        {
          fprintf (stderr, "add_at: unknown option %s\n", argv[a]);
          return 2;
        }
    }
  if (argc - a != 4)
    {
      fprintf (stderr, "usage: add_at [--snr] [--test-no-limiter] in.wav out.wav <payload hex> <zero_frames>\n");
      return 2;
    }
  const std::string infile = argv[a], outfile = argv[a + 1], bits = argv[a + 2];
  const size_t zero_frames = strtoull (argv[a + 3], nullptr, 10);

  Key key;                                       /* the zero key, as audiowmark without --key */
  Error err;
  std::unique_ptr<AudioInputStream> in_stream = AudioInputStream::create (infile, err);
  if (err)
    {
      fprintf (stderr, "add_at: error opening %s: %s\n", infile.c_str(), err.message());
      return 1;
    }
  std::unique_ptr<AudioOutputStream> out_stream = AudioOutputStream::create (outfile, in_stream->n_channels(), in_stream->sample_rate(), 16,
                                                                           Encoding::SIGNED, in_stream->n_frames(), err);
  if (err)
    {
      fprintf (stderr, "add_at: error writing to %s: %s\n", outfile.c_str(), err.message());
      return 1;
    }
  return add_stream_watermark (key, in_stream.get(), out_stream.get(), bits, zero_frames);
}
