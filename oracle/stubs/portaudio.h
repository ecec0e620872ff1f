/* oracle/stubs/portaudio.h -- declaration-only stand-in for PortAudio's header, enough for the reference's funcube.c to
 * compile into the oracle (oracle/ref_funcube.c).  TEST INFRASTRUCTURE.  Pa_ReadStream, Pa_StartStream, Pa_StopStream
 * and Pa_GetErrorText are defined by ref_funcube.c; the rest are aborting stubs (oracle/ref_iqcorr_stubs.c). */
#ifndef ORACLE_STUB_PORTAUDIO_H
#define ORACLE_STUB_PORTAUDIO_H
typedef int PaError;
typedef int PaDeviceIndex;
typedef double PaTime;
typedef unsigned long PaSampleFormat;
typedef unsigned long PaStreamFlags;
typedef void PaStream;
typedef int PaHostApiIndex;
enum PaErrorCode { paNoError = 0, paInputOverflowed = -9981 };
#define paNoDevice ((PaDeviceIndex)-1)
#define paInt16 ((PaSampleFormat)0x00000008)
#define paFramesPerBufferUnspecified (0)
#define paNoFlag ((PaStreamFlags)0)
typedef struct PaDeviceInfo {
  int structVersion;
  const char *name;
  PaHostApiIndex hostApi;
  int maxInputChannels;
  int maxOutputChannels;
  PaTime defaultLowInputLatency;
  PaTime defaultLowOutputLatency;
  PaTime defaultHighInputLatency;
  PaTime defaultHighOutputLatency;
  double defaultSampleRate;
} PaDeviceInfo;
typedef struct PaStreamParameters {
  PaDeviceIndex device;
  int channelCount;
  PaSampleFormat sampleFormat;
  PaTime suggestedLatency;
  void *hostApiSpecificStreamInfo;
} PaStreamParameters;
typedef int PaStreamCallback(const void *, void *, unsigned long, const void *, unsigned long, void *);
PaError Pa_Initialize(void);
PaError Pa_Terminate(void);
const char *Pa_GetErrorText(PaError errorCode);
PaDeviceIndex Pa_GetDeviceCount(void);
const PaDeviceInfo *Pa_GetDeviceInfo(PaDeviceIndex device);
PaError Pa_OpenStream(PaStream **stream, const PaStreamParameters *inputParameters, const PaStreamParameters *outputParameters,
                      double sampleRate, unsigned long framesPerBuffer, PaStreamFlags streamFlags,
                      PaStreamCallback *streamCallback, void *userData);
PaError Pa_StartStream(PaStream *stream);
PaError Pa_StopStream(PaStream *stream);
PaError Pa_ReadStream(PaStream *stream, void *buffer, unsigned long frames);
#endif
